"""Shutter-angle motion blur without a GPU: FrameRateConverter(shutter_angle=A, shutter_samples=S) with a stub model and the host-simulation
build of gimmvfi_op_blend_u8, against a restatement of the schedule in exact Fractions and of the blend in numpy float32: the samples each
output keeps, snapped samples, samples outside the clip, the queries sent (t strictly inside (0, 1), each pair in one call, each kept
sample queried once), bytes independent of pairs_per_call, S = 1 against shutter_angle=None, scene cuts and a one-frame shot; the op
itself bit-exact for 1 to 63 sources of both kinds, and its refusals; argument validation; the C declaration and export."""
import ctypes as C
import math
import os
import re
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

from gimmvfi_b200.video import InputPadder

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

SNAP = Fraction(1, 10 ** 6)


@pytest.fixture(scope="module")
def simlib():
    sys.path.insert(0, os.path.join(HERE, "hostsim"))
    import harness

    from gimmvfi_b200._lib import Lib

    return Lib(harness.build_hostsim())


# ------------------------------------------------------------------ the blend restated in numpy
def blend_ref(sources, top, left, h, w, bgr):
    """float32 acc = acc + v in source order (v = x * 255 for a (3,H,W) float source, the byte for an (h,w,3) uint8 one), then
    trunc(clamp(acc / n, 0, 255))"""
    acc = np.zeros((h, w, 3), np.float32)
    for s in sources:
        s = np.asarray(s)
        if s.dtype == np.float32:
            v = s[:, top:top + h, left:left + w].transpose(1, 2, 0) * np.float32(255)
        else:
            v = s.astype(np.float32)
        acc = (acc + v).astype(np.float32)
    out = np.clip(acc / np.float32(len(sources)), np.float32(0), np.float32(255)).astype(np.uint8)
    return out[..., ::-1] if bgr else out


def sim_blend(lib, sources, H, W, top, left, h, w, bgr):
    n = len(sources)
    dst = np.full((h, w, 3), 77, np.uint8)
    ptrs = (C.c_void_p * n)(*[s.ctypes.data for s in sources])
    kinds = (C.c_int * n)(*[int(s.dtype == np.float32) for s in sources])
    lib.check(lib.dll.gimmvfi_op_blend_u8(ptrs, kinds, n, H, W, top, left, C.c_void_p(dst.ctypes.data), h, w, int(bgr), None))
    return dst


def _unaligned_u8(x):
    """a copy of x that starts one byte past a 16-byte boundary"""
    buf = np.empty(x.nbytes + 32, np.uint8)
    off = (-buf.ctypes.data) % 16 + 1
    v = buf[off:off + x.nbytes].reshape(x.shape)
    v[...] = x
    return v


@pytest.mark.parametrize("h,w,top,left", [(1, 1, 0, 0), (3, 5, 1, 2), (17, 31, 7, 0), (30, 50, 1, 7), (64, 96, 0, 0), (41, 257, 3, 9)])
def test_op_matches_numpy(simlib, h, w, top, left):
    rng = np.random.default_rng(h * 1000 + w)
    H, W = h + top + 2, w + left + 3
    for n in range(1, 64):
        srcs = []
        for i in range(n):
            if rng.integers(0, 2):
                # values past [0, 1] too: the clamp
                srcs.append(rng.uniform(-0.2, 1.2, (3, H, W)).astype(np.float32))
            else:
                u = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
                srcs.append(_unaligned_u8(u) if i % 3 == 0 else u)
        for bgr in (False, True):
            got = sim_blend(simlib, srcs, H, W, top, left, h, w, bgr)
            assert np.array_equal(got, blend_ref(srcs, top, left, h, w, bgr)), (n, bgr)


def test_op_one_float_source_is_pred_to_u8(simlib):
    """n = 1: gimmvfi_op_pred_to_u8's bytes"""
    rng = np.random.default_rng(5)
    h, w, top, left, H, W = 19, 23, 2, 5, 32, 32
    x = rng.uniform(-0.1, 1.1, (1, 3, H, W)).astype(np.float32)
    for bgr in (0, 1):
        want = np.empty((1, h, w, 3), np.uint8)
        simlib.check(simlib.dll.gimmvfi_op_pred_to_u8(C.c_void_p(x.ctypes.data), 1, H, W, C.c_void_p(want.ctypes.data), h, w, top, left,
                                                      bgr, None))
        assert np.array_equal(sim_blend(simlib, [x[0]], H, W, top, left, h, w, bgr), want[0])


@pytest.mark.parametrize("n", [1, 2, 3, 7, 63])
def test_op_copies_of_one_frame_give_it_back(simlib, n):
    u = np.random.default_rng(n).integers(0, 256, (13, 29, 3), dtype=np.uint8)
    u[0, 0] = (0, 255, 254)
    assert np.array_equal(sim_blend(simlib, [u] * n, 13, 29, 0, 0, 13, 29, False), u)
    assert np.array_equal(sim_blend(simlib, [u] * n, 13, 29, 0, 0, 13, 29, True), u[..., ::-1])


def test_op_refuses_bad_arguments(simlib):
    from gimmvfi_b200._lib import GimmvfiError

    u = np.zeros((4, 4, 3), np.uint8)
    dst = np.zeros((4, 4, 3), np.uint8)

    def call(n, H=4, W=4, top=0, left=0, h=4, w=4, src=u.ctypes.data, out=dst.ctypes.data, kinds=True):
        ptrs = (C.c_void_p * 64)(*([src] * 64))
        k = (C.c_int * 64)(*([0] * 64)) if kinds else None
        return simlib.dll.gimmvfi_op_blend_u8(ptrs, k, n, H, W, top, left, C.c_void_p(out), h, w, 0, None)

    assert call(1) == 0 and call(63) == 0
    for kw in (dict(n=0), dict(n=64), dict(n=-1), dict(n=1, src=None), dict(n=1, out=None), dict(n=1, kinds=False),
               dict(n=1, h=0), dict(n=1, w=0), dict(n=1, top=1), dict(n=1, left=-1), dict(n=1, H=3), dict(n=1, h=4, w=5)):
        assert call(**kw) != 0, kw
        with pytest.raises(GimmvfiError, match="blend_u8"):
            simlib.check(call(**kw))
    assert simlib.dll.gimmvfi_op_blend_u8(None, None, 1, 4, 4, 0, 0, C.c_void_p(dst.ctypes.data), 4, 4, 0, None) != 0


def test_blend_is_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "gimmvfi_b200.h")).read()
    assert re.search(r"\bint gimmvfi_op_blend_u8\(const void\* const\* src, const int\* is_f32, int n, int H, int W, int pad_top, "
                     r"int pad_left, uint8_t\* dst, int h, int w,\s+int bgr, void\* stream\);", header)
    from gimmvfi_b200._lib import EXPORTS, default_lib

    assert "gimmvfi_op_blend_u8" in EXPORTS
    assert getattr(default_lib().dll, "gimmvfi_op_blend_u8") is not None


# ------------------------------------------------------------------ the converter with a stub model and the host-simulation op
h, w = 30, 50      # padded to 32 x 64 at (1, 7): the crop matters


def _pad(u8):
    """InputPadder.pad_u8 on the host: (n,h,w,3) uint8 -> (n,3,H,W) float32 / 255, replicate-padded"""
    p = InputPadder((h, w), 32)._pad
    x = u8.permute(0, 3, 1, 2).to(torch.float32) / 255.0
    return torch.nn.functional.pad(x, p, mode="replicate")


class _Padder:
    """InputPadder's arithmetic on host tensors; unpad_u8 is pred_to_u8's trunc(clamp(x * 255)) in float32"""

    def __init__(self, dims, divisor=32):
        self._p = InputPadder(dims, divisor)
        self.ht, self.wd, self.padded_shape = self._p.ht, self._p.wd, self._p.padded_shape

    def unpad_box(self, ht, wd):
        return self._p.unpad_box(ht, wd)

    def pad_u8(self, f):
        return _pad(f)

    def unpad_u8(self, pred, bgr=True):
        top, bottom, left, right = self.unpad_box(*pred.shape[-2:])
        out = (pred * 255.0).clamp(0, 255).to(torch.uint8)[:, :, top:bottom, left:right].permute(0, 2, 3, 1).contiguous()
        return out.flip(-1) if bgr else out


def _frame(j):
    """input frame j: seeded noise, with j at pixel (0, 0) channel 0 (so the padded corner names the frame)"""
    g = torch.Generator().manual_seed(1000 + j)
    f = torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, generator=g)
    f[0, 0, 0] = j
    return f


def _index(padded):
    return int(round(padded[0, 0, 0].item() * 255))


def _mix(a, b, t):
    return a * (1 - t) + b * t


class _Stub:
    """interpolate_at as the t-weighted mix of the two padded frames; records every call's queries by input frame index"""

    tensor_cores = 4

    def __init__(self):
        self.calls = []

    def _interpolate_at(self, frames, queries, ds, aux):
        assert aux is False
        self.calls.append([(_index(frames[a]), _index(frames[b]), t) for a, b, t in queries])
        return {"imgt_pred": torch.stack([_mix(frames[a], frames[b], t) for a, b, t in queries], 0)}


@pytest.fixture
def V(monkeypatch, simlib):
    import gimmvfi_b200.video as V

    monkeypatch.setattr(V, "InputPadder", _Padder)
    monkeypatch.setattr(V, "default_lib", lambda: simlib)
    return V


def _shot(f, cuts):
    return sum(1 for c in cuts if c <= f)


def schedule(fps_in, fps_out, n, A, S, cuts=(), beyond=Fraction(0)):
    """the outputs of n frames, each [(instant, source)] over its kept samples in order, source ("frame", f) or ("query", a, a + 1, t);
    with `beyond`, also the samples of outputs up to that far past the last frame, and none dropped (every query that may be sent)"""
    step = Fraction(fps_in) / Fraction(fps_out)
    wnd = Fraction(A) / 360 * step
    last = n - 1
    outs, k = [], 0
    while k * step <= last + beyond:
        tau = k * step
        samples, own = [], None
        for i in range(S):
            x = tau - wnd / 2 + Fraction(2 * i + 1, 2 * S) * wnd
            if (x < 0 or x > last) and not beyond:
                continue
            a = math.floor(x)
            off = x - a
            if off <= SNAP:
                src = ("frame", a)
            elif off >= 1 - SNAP:
                src = ("frame", a + 1)
            elif a + 1 in cuts:
                src = ("frame", a if off <= Fraction(1, 2) else a + 1)
            else:
                src = ("query", a, a + 1, float(np.float32(float(off))))
            samples.append((x, src))
            if x == tau:
                own = src
        assert own is not None or beyond
        if not beyond:
            shot = _shot(own[1], cuts)
            samples = [(x, s) for x, s in samples if _shot(s[1], cuts) == shot]
        outs.append(samples)
        k += 1
    return outs


def expected_bytes(sched, bgr=True):
    top, _, left, _ = InputPadder((h, w), 32).unpad_box(*InputPadder((h, w), 32).padded_shape)
    out = []
    for samples in sched:
        srcs = []
        for _, s in samples:
            if s[0] == "frame":
                srcs.append(_frame(s[1]).numpy())
            else:
                pa, pb = _pad(torch.stack([_frame(s[1]), _frame(s[2])], 0))
                srcs.append(_mix(pa, pb, s[3]).numpy())
        out.append(torch.from_numpy(np.ascontiguousarray(blend_ref(srcs, top, left, h, w, bgr))))
    return out


def run(V, fps_in, fps_out, n, K, A=None, S=7, bgr=True, threshold=None):
    m = _Stub()
    conv = V.FrameRateConverter(m, fps_in, fps_out, bgr=bgr, pairs_per_call=K, shutter_angle=A, shutter_samples=S,
                                scene_threshold=threshold)
    out = []
    for j in range(n):
        got = conv.push(_frame(j))
        assert all(o.shape == (h, w, 3) and o.dtype == torch.uint8 for o in got)
        out += got
    out += conv.flush()
    return m, conv, out


RATES = [(60, 24), (24, 60), ("30000/1001", 24), (50, 25), (30, 30)]
N = 16


def check_calls(calls, sched, fps_in, fps_out, A, S, cuts=()):
    """the queries sent: each pair in one call and never a cut, every t strictly inside (0, 1) and the float32 offset of a sample, every
    kept interpolated sample queried exactly once"""
    every = {s[1:] for out in schedule(fps_in, fps_out, N, A, S, cuts, beyond=Fraction(fps_in) / Fraction(fps_out)) for _, s in out
             if s[0] == "query"}
    where = {}
    for c, qs in enumerate(calls):
        for a, b, t in qs:
            assert b == a + 1 and 0.0 < t < 1.0 and (a, b, t) in every, (a, b, t)
            assert b not in cuts
            where.setdefault((a, b), set()).add(c)
    assert all(len(v) == 1 for v in where.values()), where
    sent = [q for qs in calls for q in qs]
    for out in sched:
        for _, s in out:
            if s[0] == "query":
                assert sent.count(s[1:]) == 1, s


@pytest.mark.parametrize("S", [1, 3, 5, 7])
@pytest.mark.parametrize("A", [90, 180, 360])
@pytest.mark.parametrize("fps_in,fps_out", RATES)
def test_schedule_and_bytes(V, fps_in, fps_out, A, S):
    sched = schedule(fps_in, fps_out, N, A, S)
    want = expected_bytes(sched)
    got = {}
    for K in (1, 3):
        m, conv, out = run(V, fps_in, fps_out, N, K, A, S)
        assert len(out) == len(sched)
        for k, (o, e) in enumerate(zip(out, want)):
            assert torch.equal(o, e), (K, k, sched[k])
        check_calls(m.calls, sched, fps_in, fps_out, A, S)
        assert all(len({(a, b) for a, b, _ in qs}) <= K for qs in m.calls)
        got[K] = out
    assert all(torch.equal(a, b) for a, b in zip(got[1], got[3]))
    # the samples dropped at the ends of the clip
    step = Fraction(fps_in) / Fraction(fps_out)
    wnd = Fraction(A) / 360 * step
    for k, out in enumerate(sched):
        inside = [i for i in range(S) if 0 <= k * step - wnd / 2 + Fraction(2 * i + 1, 2 * S) * wnd <= N - 1]
        assert len(out) == len(inside) and (k * step - wnd / 2 >= 0 and k * step + wnd / 2 <= N - 1) <= (len(out) == S)


@pytest.mark.parametrize("bgr", [True, False])
@pytest.mark.parametrize("fps_in,fps_out", RATES)
def test_one_sample_is_no_shutter(V, fps_in, fps_out, bgr):
    """S = 1 gives the bytes, the engine calls and the per-push returns of shutter_angle=None"""
    for K in (1, 3):
        for A in (90, 360):
            ref_m, _, ref = run(V, fps_in, fps_out, N, K, bgr=bgr)
            m, _, out = run(V, fps_in, fps_out, N, K, A, 1, bgr=bgr)
            assert m.calls == ref_m.calls
            assert len(out) == len(ref) and all(torch.equal(a, b) for a, b in zip(out, ref))


def test_none_makes_no_blend(V, monkeypatch):
    def boom(*a, **k):
        raise AssertionError("blend_u8 was called")

    monkeypatch.setattr(V, "blend_u8", boom)
    run(V, 60, 24, N, 2)


def _patch_scores(V, monkeypatch, scores):
    """pair (j - 1, j) scores scores.get(j, 5.0)"""
    def pair_sums(a, b):
        j = int(b[0, 0, 0])
        assert int(a[0, 0, 0]) == j - 1
        return torch.tensor([[round(scores.get(j, 5.0) * 3 * h * w), 0, 0]], dtype=torch.int64)

    monkeypatch.setattr(V, "_pair_sums", pair_sums)


@pytest.mark.parametrize("K", [1, 3])
@pytest.mark.parametrize("fps_in,fps_out,A,S", [(60, 24, 360, 7), (60, 24, 180, 5), (24, 60, 360, 3), (120, 24, 360, 7), (30, 30, 270, 5)])
def test_cuts(V, monkeypatch, fps_in, fps_out, A, S, K):
    """cuts at 4, 5 and 9: no query for a cut pair, and each output keeps only the samples of its own shot"""
    cuts = (4, 5, 9)
    _patch_scores(V, monkeypatch, {c: 50.0 for c in cuts})
    m, conv, out = run(V, fps_in, fps_out, N, K, A, S, threshold=27)
    assert conv.cuts == list(cuts)
    sched = schedule(fps_in, fps_out, N, A, S, cuts)
    for k, (o, e) in enumerate(zip(out, expected_bytes(sched))):
        assert torch.equal(o, e), (k, sched[k])
    assert len(out) == len(sched)
    check_calls(m.calls, sched, fps_in, fps_out, A, S, cuts)
    for samples in sched:   # each output within one shot
        assert len({_shot(s[1], cuts) for _, s in samples}) == 1


def test_one_frame_shot(V, monkeypatch):
    """120 -> 24 at 360 degrees, S = 3, frame 10 a shot of its own (cuts at 10 and 11): output 2 (tau = 10) keeps only its middle sample,
    and is frame 10"""
    _patch_scores(V, monkeypatch, {10: 60.0, 11: 60.0})
    m, conv, out = run(V, 120, 24, N, 1, 360, 3, threshold=27)
    assert conv.cuts == [10, 11]
    assert torch.equal(out[2], _frame(10).flip(-1))
    assert schedule(120, 24, N, 360, 3, (10, 11))[2] == [(10, ("frame", 10))]
    assert not any(b in (10, 11) for qs in m.calls for _, b, _ in qs)


def test_flush_ends_the_clip(V):
    m = _Stub()
    conv = V.FrameRateConverter(m, 60, 24, shutter_angle=180, shutter_samples=3)
    first = []
    for j in range(N):
        first += conv.push(_frame(j))
    first += conv.flush()
    again = []
    for j in range(N):
        again += conv.push(_frame(j))
    again += conv.flush()
    assert len(first) == len(again) and all(torch.equal(a, b) for a, b in zip(first, again))


@pytest.mark.parametrize("bad", [0, -90, 360.5, 361, float("nan"), float("inf"), True, "180", None])
def test_bad_angles_are_refused(bad):
    from gimmvfi_b200.video import FrameRateConverter

    if bad is None:
        assert FrameRateConverter(_Stub(), 60, 24, shutter_angle=None).window is None
        return
    with pytest.raises(ValueError, match="shutter_angle"):
        FrameRateConverter(_Stub(), 60, 24, shutter_angle=bad)


@pytest.mark.parametrize("bad", [0, 2, 65, 2.5, True, -1, 64, "7", 7.0])
def test_bad_sample_counts_are_refused(bad):
    from gimmvfi_b200.video import FrameRateConverter

    with pytest.raises(ValueError, match="shutter_samples"):
        FrameRateConverter(_Stub(), 60, 24, shutter_angle=180, shutter_samples=bad)


def test_angles_are_exact():
    from gimmvfi_b200.video import FrameRateConverter

    c = FrameRateConverter(_Stub(), 60, 24, shutter_angle=172.8, shutter_samples=63)
    assert c.shutter_angle == Fraction(864, 5) and c.window == Fraction(864, 5) / 360 * Fraction(5, 2)
    assert FrameRateConverter(_Stub(), 60, 24, shutter_angle=np.int64(360), shutter_samples=np.int32(1)).window == Fraction(5, 2)


@pytest.mark.parametrize("fps_in,fps_out,A,S", [(120, 24, 360, 5), (60, 20, 360, 3)])
def test_windows_of_input_frames_stream_with_cuts(V, monkeypatch, fps_in, fps_out, A, S):
    """every sample falls on an input frame, so no engine call is ever made: with scene cuts on, each output still comes back from the
    push that completes its window (its scores are read back then), and nothing piles up in the queue"""
    n, cuts = 60, (23, 41)
    _patch_scores(V, monkeypatch, {c: 50.0 for c in cuts})
    m = _Stub()
    conv = V.FrameRateConverter(m, fps_in, fps_out, pairs_per_call=2, shutter_angle=A, shutter_samples=S, scene_threshold=27)
    sched = schedule(fps_in, fps_out, n, A, S, cuts)
    assert all(s[0] == "frame" for out in sched for _, s in out)
    step = Fraction(fps_in) / Fraction(fps_out)
    wnd = Fraction(A) / 360 * step
    out = []
    for j in range(n):
        got = conv.push(_frame(j))
        out += got
        # every output whose window ends by frame j has come back
        assert len(out) == sum(1 for k in range(len(sched)) if k * step + wnd / 2 - wnd / (2 * S) <= j), j
        assert len(conv._queue) <= 2, j
    out += conv.flush()
    assert m.calls == [] and conv.cuts == list(cuts)
    assert len(out) == len(sched) and all(torch.equal(o, e) for o, e in zip(out, expected_bytes(sched)))


def test_waiting_outputs_keep_copies_of_their_sub_frames(V):
    """an output still waiting after an engine call holds clones of its sub-frames, not views that keep the call's whole output alive"""
    conv = V.FrameRateConverter(_Stub(), 60, 24, pairs_per_call=3, shutter_angle=360, shutter_samples=7)
    held = 0
    for j in range(N):
        conv.push(_frame(j))
        for e in conv._queue:
            for s in e.samples:
                if s.out is not None:
                    held += 1
                    assert s.out._base is None and s.out.shape == (3, 32, 64)
    assert held > 0
    conv.flush()
