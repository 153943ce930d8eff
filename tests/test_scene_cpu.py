"""Scene-cut detection without a GPU: the host-simulation build of gimmvfi_op_scene_sums against cv2's RGB -> HSV (every 8-bit colour, and
random frames up to 1080x1920), the C export, and FrameRateConverter / VideoInterpolator with chosen scores and stub models: no engine work
for a cut, the nearer input frame in its place, K grouping, `cuts`, when the K = 1 frame cache is loaded, and scene_threshold=None
unchanged."""
import ctypes as C
import math
import os
import re
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# ------------------------------------------------------------------ the op, host simulation
@pytest.fixture(scope="module")
def simlib():
    sys.path.insert(0, os.path.join(HERE, "hostsim"))
    import harness

    from gimmvfi_b200._lib import Lib

    return Lib(harness.build_hostsim())


def sim_sums(lib, a, b):
    """the op on two (n,h,w,3) uint8 numpy stacks -> (n,3) uint64"""
    n, h, w, _ = a.shape
    sums = np.full((n, 3), 0xDEADBEEF, np.uint64)   # every sum must be written
    lib.check(lib.dll.gimmvfi_op_scene_sums(C.c_void_p(a.ctypes.data), C.c_void_p(b.ctypes.data), n, h, w, C.c_void_p(sums.ctypes.data), None))
    return sums


def hsv_restated(x):
    """the integer RGB -> HSV of the op, restated in numpy: (..., 3) uint8 -> (..., 3) int64"""
    x = x.astype(np.int64)
    r, g, b = x[..., 0], x[..., 1], x[..., 2]
    v = x.max(-1)
    d = v - x.min(-1)
    idx = np.arange(256)
    sdiv = np.where(idx > 0, (2 * 255 * 4096 + idx) // np.maximum(2 * idx, 1), 0)
    hdiv = np.where(idx > 0, (2 * 180 * 4096 + 6 * idx) // np.maximum(12 * idx, 1), 0)
    s = (d * sdiv[v] + 2048) >> 12
    h0 = np.where(v == r, g - b, np.where(v == g, b - r + 2 * d, r - g + 4 * d))
    h = (h0 * hdiv[d] + 2048) >> 12
    h = np.where(h < 0, h + 180, h)
    return np.stack([h, s, v], -1)


def cv2_sums(a, b):
    cv2 = pytest.importorskip("cv2")
    hsv = lambda x: cv2.cvtColor(np.ascontiguousarray(x), cv2.COLOR_RGB2HSV).astype(np.int64)
    return np.stack([np.abs(hsv(x) - hsv(y)).reshape(-1, 3).sum(0) for x, y in zip(a, b)], 0)


def test_every_colour_against_cv2(simlib):
    """2^24 pairs of 1x1 frames: every RGB colour against black, whose HSV is (0, 0, 0) -> the colour's H + S + V"""
    cv2 = pytest.importorskip("cv2")
    c = np.arange(1 << 24, dtype=np.uint32)
    a = np.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).astype(np.uint8).reshape(-1, 1, 1, 3)
    b = np.zeros_like(a)
    got = sim_sums(simlib, a, b).astype(np.int64)
    want = cv2.cvtColor(a.reshape(4096, 4096, 3), cv2.COLOR_RGB2HSV).reshape(-1, 3).astype(np.int64)
    assert np.array_equal(got, want), np.argwhere(got != want)[:5]
    assert np.array_equal(hsv_restated(a.reshape(-1, 3)), want)


@pytest.mark.parametrize("size", [(1, 1), (17, 31), (120, 150), (1080, 1920)])
def test_scores_against_cv2_on_random_frames(simlib, size):
    from gimmvfi_b200.video import scores_from_sums

    h, w = size
    rng = np.random.default_rng(h * 7919 + w)
    frames = rng.integers(0, 256, (6, h, w, 3), dtype=np.uint8)
    frames[3] = frames[2] // 2 + 40    # a pair of related frames besides the unrelated ones
    for n in range(1, 6):
        a, b = frames[:n], frames[1:n + 1]
        got = sim_sums(simlib, a, b)
        want = cv2_sums(a, b)
        assert np.array_equal(got.astype(np.int64), want), (size, n)
        scores = scores_from_sums(torch.from_numpy(got.astype(np.int64)), h, w)
        ref = want.sum(1).astype(np.float64) / (3 * h * w)
        assert scores.dtype == torch.float64 and np.array_equal(scores.numpy(), ref), (size, n)


def test_sums_refuse_bad_sizes(simlib):
    from gimmvfi_b200._lib import GimmvfiError

    a = np.zeros((1, 2, 2, 3), np.uint8)
    s = np.zeros((1, 3), np.uint64)
    for n, h, w in ((-1, 2, 2), (1, 0, 2), (1, 2, 0), (1, 1 << 16, 1 << 15)):
        with pytest.raises(GimmvfiError, match="scene_sums"):
            simlib.check(simlib.dll.gimmvfi_op_scene_sums(C.c_void_p(a.ctypes.data), C.c_void_p(a.ctypes.data), n, h, w,
                                                          C.c_void_p(s.ctypes.data), None))


def test_scene_sums_is_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "gimmvfi_b200.h")).read()
    assert re.search(r"\bint gimmvfi_op_scene_sums\(const uint8_t\* a, const uint8_t\* b, int n, int h, int w, uint64_t\* sums", header)
    from gimmvfi_b200._lib import EXPORTS, default_lib

    assert "gimmvfi_op_scene_sums" in EXPORTS
    assert getattr(default_lib().dll, "gimmvfi_op_scene_sums") is not None


def test_scene_scores_refuses_host_tensors():
    from gimmvfi_b200.video import scene_scores

    with pytest.raises(ValueError, match="CUDA"):
        scene_scores(torch.zeros(3, 4, 4, 3, dtype=torch.uint8))
    with pytest.raises(ValueError, match="CUDA"):
        scene_scores(np.zeros((3, 4, 4, 3), np.uint8))


# ------------------------------------------------------------------ the video classes with chosen scores and stub models
H, W = 32, 64


class _Padder:
    """InputPadder on the host: (n,h,w,3) uint8 -> (n,3,h,w) float and back (the stub frames need no padding)"""

    def __init__(self, dims, divisor=32):
        self.ht, self.wd = dims[-2:]
        self.padded_shape = (self.ht, self.wd)

    def pad_u8(self, f):
        return f.permute(0, 3, 1, 2).to(torch.float32) / 255.0

    def unpad_u8(self, pred, bgr=True):
        out = (pred * 255.0).round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1)
        return out.flip(-1) if bgr else out


def _frame(j):
    """input frame j: channel c holds 10 j + c, so a frame's index can be read back and a BGR flip is visible"""
    f = torch.zeros(H, W, 3, dtype=torch.uint8)
    for c in range(3):
        f[..., c] = 10 * j + c
    return f


def _index(f):
    """the input index of a padded float frame (3,h,w)"""
    return int(round(f[0, 0, 0].item() * 255)) // 10


def _u8_index(f):
    return int(f[0, 0, 0].item()) // 10


def _mix(a, b, t):
    return (1 - t) * a + t * b


class _StubModel:
    """interpolates by the weighted mean of the two frames, with a flow of value t; records every call by input frame index"""

    tensor_cores = 4

    def __init__(self):
        self.calls = []
        self.engine = types.SimpleNamespace(frame_cache_bytes=lambda *a: 16, weights_version=0)

    def sample_coord_input(self, B, shape, ts, device=None, upsample_ratio=1.0):
        return torch.zeros(B, 1, int(shape[0] * upsample_ratio), int(shape[1] * upsample_ratio), 3)

    def _interpolate_at(self, frames, queries, ds, aux):
        assert aux is False
        self.calls.append(("queries", [(_index(frames[a]), _index(frames[b]), t) for a, b, t in queries], frames.shape[0]))
        return {"imgt_pred": torch.stack([_mix(frames[a], frames[b], t) for a, b, t in queries], 0)}

    def _interpolate(self, xs, coords, ts, ds, aux, frame_cache=None):
        a, b = xs[0, :, 0], xs[0, :, 1]
        self.calls.append(("pair", (_index(a), _index(b)), frame_cache[1]))
        out = {"imgt_pred": [_mix(a, b, float(t[0])).unsqueeze(0) for t in ts]}
        if aux:
            out["flowt"] = [torch.full((2, H, W), float(t[0])) for t in ts]
        return out

    def _interpolate_clip(self, frames, pairs, t, ds, aux):
        self.calls.append(("clip", [(_index(frames[a]), _index(frames[b])) for a, b in pairs], frames.shape[0]))
        out = {"imgt_pred": [torch.stack([_mix(frames[a], frames[b], ti) for a, b in pairs], 0) for ti in t]}
        if aux:   # forward's .squeeze() of a single pair
            out["flowt"] = [torch.full((len(pairs), 2, H, W), ti).squeeze() for ti in t]
        return out


class _Scores:
    """the score source: pair (j - 1, j) scores scores.get(j, 5.0); records the pairs scored and the reads back"""

    def __init__(self, V, monkeypatch, scores):
        self.scores, self.pairs, self.reads = scores, [], 0
        read = V.scores_from_sums

        def pair_sums(a, b):
            j = _u8_index(b)
            assert _u8_index(a) == j - 1
            self.pairs.append(j)
            return torch.tensor([[round(self.scores.get(j, 5.0) * 3 * H * W), 0, 0]], dtype=torch.int64)

        def counted(sums, h, w):
            self.reads += 1
            return read(sums, h, w)

        monkeypatch.setattr(V, "_pair_sums", pair_sums)
        monkeypatch.setattr(V, "scores_from_sums", counted)


@pytest.fixture
def V(monkeypatch):
    import gimmvfi_b200.video as V

    monkeypatch.setattr(V, "InputPadder", _Padder)
    monkeypatch.setattr(V, "flow_images", lambda padder, flows, bgr: [f.clone() for f in flows])
    return V


@pytest.fixture
def no_op(V, monkeypatch):
    """scene_threshold=None must never reach the score op"""
    def boom(*a, **k):
        raise AssertionError("the score op was used")

    for name in ("_pair_sums", "_scene_sums", "scene_scores", "scores_from_sums"):
        monkeypatch.setattr(V, name, boom)
    return V


def _run_converter(V, fps_in, fps_out, n, K, threshold=None):
    m = _StubModel()
    conv = V.FrameRateConverter(m, fps_in, fps_out, pairs_per_call=K, scene_threshold=threshold)
    out = []
    for j in range(n):
        out += conv.push(_frame(j))
    out += conv.flush()
    return m, conv, out


def _sent_pairs(calls):
    return [{(a, b) for a, b, _ in qs} for kind, qs, _ in calls]


@pytest.mark.parametrize("K", [1, 2, 4])
@pytest.mark.parametrize("fps_in,fps_out", [(24, 60), (24, 48), (60, 24), (25, 30)])
def test_converter_skips_cuts(V, monkeypatch, fps_in, fps_out, K):
    """cuts at 3, 4 (two in a row) and 8: no query for them, the nearer input frame at each of their instants (ties to the earlier),
    every other output as without a threshold, at most K pairs per call, one read back per call or flush"""
    from fractions import Fraction

    n = 12
    ref_m, _, ref = _run_converter(V, fps_in, fps_out, n, K)
    sc = _Scores(V, monkeypatch, {3: 40.0, 4: 27.0, 8: 90.0, 6: 26.999})
    m, conv, out = _run_converter(V, fps_in, fps_out, n, K, threshold=27)
    assert conv.cuts == [3, 4, 8]
    assert sc.pairs == list(range(1, n))
    assert len(out) == len(ref)
    step = Fraction(fps_in, fps_out)
    for k, (o, r) in enumerate(zip(out, ref)):
        tau = k * step
        j = math.ceil(tau)
        off = tau - (j - 1)
        if tau.denominator != 1 and j in conv.cuts:
            assert torch.equal(o, _frame(j - 1 if off <= Fraction(1, 2) else j).flip(-1)), k
        else:
            assert torch.equal(o, r), k
    sent = _sent_pairs(m.calls)
    assert all(1 <= len(p) <= K for p in sent)
    assert not any(b in conv.cuts for p in sent for _, b in p)
    want = [q for _, qs, _ in ref_m.calls for q in qs if q[1] not in conv.cuts]
    assert [q for _, qs, _ in m.calls for q in qs] == want
    for (_, qs, nf) in m.calls:   # only the frames of the pairs sent
        assert nf == len({f for a, b, _ in qs for f in (a, b)})
    assert sc.reads <= len(ref_m.calls) + 1   # one per block of K pairs with queries, sent or not, and the final flush


def test_converter_all_cut_block_makes_no_call(V, monkeypatch):
    """24 -> 60 with K = 2: pairs (0,1), (1,2) go in one call, (2,3), (3,4) are both cuts: no call for them"""
    ref_m, _, _ = _run_converter(V, 24, 60, 7, 2)
    _Scores(V, monkeypatch, {3: 50.0, 4: 50.0})
    m, conv, out = _run_converter(V, 24, 60, 7, 2, threshold=27)
    assert _sent_pairs(ref_m.calls) == [{(0, 1), (1, 2)}, {(2, 3), (3, 4)}, {(4, 5), (5, 6)}]
    assert _sent_pairs(m.calls) == [{(0, 1), (1, 2)}, {(4, 5), (5, 6)}]
    assert conv.cuts == [3, 4]


def test_converter_none_is_unchanged(no_op):
    """without a threshold the score op is never touched, and a threshold no pair reaches gives the same calls and outputs"""
    V = no_op
    m, conv, out = _run_converter(V, 24, 60, 9, 3)
    assert conv.cuts == []
    assert _sent_pairs(m.calls) == [{(0, 1), (1, 2), (2, 3)}, {(3, 4), (4, 5), (5, 6)}, {(6, 7), (7, 8)}]


def test_converter_threshold_without_cuts_matches_none(V, monkeypatch):
    ref_m, _, ref = _run_converter(V, 24, 60, 9, 3)
    _Scores(V, monkeypatch, {})
    m, conv, out = _run_converter(V, 24, 60, 9, 3, threshold=27)
    assert m.calls == ref_m.calls and len(out) == len(ref) and all(torch.equal(a, b) for a, b in zip(out, ref))


def test_converter_reset_starts_a_new_clip(V, monkeypatch):
    sc = _Scores(V, monkeypatch, {2: 50.0})
    conv = V.FrameRateConverter(_StubModel(), 24, 60, scene_threshold=27)
    for j in range(4):
        conv.push(_frame(j))
    conv.flush()
    assert conv.cuts == [2]
    conv.reset()
    assert conv.cuts == []
    conv.push(_frame(5))
    assert sc.pairs == [1, 2, 3]    # no score across the reset


def _run_vi(V, N, K, n, threshold=None, with_flow=False, bgr=True):
    m = _StubModel()
    vi = V.VideoInterpolator(m, N=N, pairs_per_call=K, scene_threshold=threshold, with_flow=with_flow, bgr=bgr)
    frames, flows = [], []
    for j in range(n):
        got = vi.push(_frame(j))
        f, fl = got if with_flow else (got, [])
        frames += f
        flows += fl
    got = vi.flush()
    f, fl = got if with_flow else (got, [])
    return m, vi, frames + f, flows + fl


@pytest.mark.parametrize("with_flow", [False, True])
@pytest.mark.parametrize("bgr", [True, False])
@pytest.mark.parametrize("K", [1, 3])
@pytest.mark.parametrize("N", [2, 4, 5])
def test_interpolator_skips_cuts(V, monkeypatch, N, K, bgr, with_flow):
    """cuts at 2, 4, 5 and 6 over 10 frames (with K = 3 the block of pairs 4..6 is all cuts): the N - 1 frames of a cut are the nearer
    input frame (t = i / N <= 1/2: the earlier), with zero flows; the others as without a threshold"""
    n, cuts = 10, [2, 4, 5, 6]
    ref_m, _, ref, ref_fl = _run_vi(V, N, K, n, with_flow=with_flow, bgr=bgr)
    sc = _Scores(V, monkeypatch, {j: 30.0 for j in cuts})
    m, vi, out, fl = _run_vi(V, N, K, n, threshold=27, with_flow=with_flow, bgr=bgr)
    assert vi.cuts == cuts and sc.pairs == list(range(1, n))
    assert len(out) == len(ref) == (n - 1) * (N - 1)
    assert len(fl) == (len(out) if with_flow else 0)
    for p in range(n - 1):
        j = p + 1
        for i in range(1, N):
            k = p * (N - 1) + i - 1
            if j in cuts:
                near = _frame(j - 1 if 2 * i <= N else j)
                assert torch.equal(out[k], near.flip(-1) if bgr else near), (j, i)
                if with_flow:
                    assert fl[k].shape == (2, H, W) and not fl[k].any(), (j, i)
            else:
                assert torch.equal(out[k], ref[k]), (j, i)
                if with_flow:
                    assert torch.equal(fl[k], ref_fl[k]), (j, i)
    if K == 1:
        assert [c[1] for c in m.calls] == [(j - 1, j) for j in range(1, n) if j not in cuts]
        # the frame cache: the first call and the one after each cut load nothing
        assert [c[2] for c in m.calls] == [False, False, False, True, True]   # pairs (0,1), (2,3), (6,7), (7,8), (8,9)
        assert sc.reads == n - 1
    else:
        assert [c[1] for c in m.calls] == [[(0, 1), (2, 3)], [(6, 7), (7, 8), (8, 9)]]
        assert [c[2] for c in m.calls] == [4, 4]
        assert sc.reads == 3


def test_interpolator_none_is_unchanged(no_op):
    for K in (1, 3):
        m, vi, out, fl = _run_vi(no_op, 3, K, 8, with_flow=True)
        assert vi.cuts == [] and len(out) == len(fl) == 7 * 2
        if K == 1:
            assert [c[1:] for c in m.calls] == [((j - 1, j), j > 1) for j in range(1, 8)]
        else:
            assert [c[1:] for c in m.calls] == [([(0, 1), (1, 2), (2, 3)], 4), ([(3, 4), (4, 5), (5, 6)], 4), ([(6, 7)], 2)]


@pytest.mark.parametrize("K", [1, 3])
def test_interpolator_threshold_without_cuts_matches_none(V, monkeypatch, K):
    ref_m, _, ref, ref_fl = _run_vi(V, 4, K, 8, with_flow=True)
    _Scores(V, monkeypatch, {})
    m, vi, out, fl = _run_vi(V, 4, K, 8, threshold=27, with_flow=True)
    assert m.calls == ref_m.calls
    assert all(torch.equal(a, b) for a, b in zip(out + fl, ref + ref_fl)) and len(out + fl) == len(ref + ref_fl)


class _FailingModel(_StubModel):
    """_StubModel whose calls with the given numbers (counted from 0) raise the given exception after they are recorded"""

    def __init__(self, fail):
        super().__init__()
        self.fail = fail

    def _interpolate(self, xs, coords, ts, ds, aux, frame_cache=None):
        out = super()._interpolate(xs, coords, ts, ds, aux, frame_cache)
        if len(self.calls) - 1 in self.fail:
            raise self.fail[len(self.calls) - 1]
        return out


def _push_all(vi, frames):
    for j in frames:
        vi.push(_frame(j))


def test_interpolator_retries_a_refused_cache_load_once(V):
    """the engine refuses the load of pair (1,2): one full forward of that pair, and the next pair loads again"""
    from gimmvfi_b200._lib import GimmvfiError

    m = _FailingModel({1: GimmvfiError("frame cache: the buffer holds another problem size")})
    vi = V.VideoInterpolator(m, N=2)
    _push_all(vi, range(4))
    assert [c[1:] for c in m.calls] == [((0, 1), False), ((1, 2), True), ((1, 2), False), ((2, 3), True)]
    # a refusal of the full forward too is not retried again
    m = _FailingModel({1: GimmvfiError("frame cache: refused"), 2: GimmvfiError("frame cache: refused")})
    vi = V.VideoInterpolator(m, N=2)
    _push_all(vi, range(2))
    with pytest.raises(GimmvfiError):
        vi.push(_frame(2))
    assert [c[1:] for c in m.calls] == [((0, 1), False), ((1, 2), True), ((1, 2), False)]


@pytest.mark.parametrize("change", ["tensor_cores", "weights_version"])
def test_interpolator_cache_not_loaded_after_a_precision_or_weights_change(V, change):
    m = _StubModel()
    vi = V.VideoInterpolator(m, N=2)
    _push_all(vi, range(3))
    if change == "tensor_cores":
        m.tensor_cores = 1
    else:
        m.engine.weights_version = 1
    _push_all(vi, range(3, 5))
    assert [c[1:] for c in m.calls] == [((0, 1), False), ((1, 2), True), ((2, 3), False), ((3, 4), True)]


def test_interpolator_cache_not_loaded_after_an_engine_error(V):
    """pair (2,3) fails: the next pair does not load, and the clip goes on from frame 3"""
    m = _FailingModel({2: RuntimeError("engine failure")})
    vi = V.VideoInterpolator(m, N=2)
    _push_all(vi, range(3))
    with pytest.raises(RuntimeError, match="engine failure"):
        vi.push(_frame(3))
    _push_all(vi, range(4, 6))
    assert [c[1:] for c in m.calls] == [((0, 1), False), ((1, 2), True), ((2, 3), True), ((3, 4), False), ((4, 5), True)]


def test_interpolator_frame_size_change_starts_a_new_clip(V, monkeypatch):
    sc = _Scores(V, monkeypatch, {1: 50.0})
    vi = V.VideoInterpolator(_StubModel(), N=2, scene_threshold=27)
    vi.push(_frame(0))
    vi.push(_frame(1))
    assert vi.cuts == [1]
    vi.push(_frame(2)[:16])
    assert vi.cuts == [] and sc.pairs == [1]


@pytest.mark.parametrize("bad", [0, -1, 0.0, float("nan"), float("inf"), -float("inf"), "27", True, [27]])
def test_bad_thresholds_are_refused(bad):
    from gimmvfi_b200.video import FrameRateConverter, VideoInterpolator

    with pytest.raises(ValueError, match="scene_threshold"):
        FrameRateConverter(_StubModel(), 24, 60, scene_threshold=bad)
    with pytest.raises(ValueError, match="scene_threshold"):
        VideoInterpolator(_StubModel(), N=2, scene_threshold=bad)


@pytest.mark.parametrize("good", [27, 27.5, np.float32(12.0), 1e-9])
def test_good_thresholds_are_kept(good):
    from gimmvfi_b200.video import FrameRateConverter, VideoInterpolator

    assert FrameRateConverter(_StubModel(), 24, 60, scene_threshold=good).scene_threshold == float(good)
    assert VideoInterpolator(_StubModel(), N=2, scene_threshold=good).scene_threshold == float(good)
