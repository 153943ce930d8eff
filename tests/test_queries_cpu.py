"""The query form of GIMM-VFI-R / -F without a GPU: interpolate_at's argument checks, the C exports, FrameRateConverter's schedule with a
stub model, and the host simulation of the engine running a query list against per-pair forwards at each pair's own timesteps."""
import math
import os
import re
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

from gimmvfi_b200.synth import synth_batch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


# ------------------------------------------------------------------ argument checks
@pytest.fixture(scope="module")
def model_r():
    from gimmvfi_b200.model import GIMMVFI_R

    return GIMMVFI_R()


@pytest.mark.parametrize("queries,match", [
    ([], "empty"),
    ([(0, 3, 0.5)], "outside"),
    ([(-1, 0, 0.5)], "outside"),
    ([(0, 1, 0.5), (2, 1, 0.5)], "outside"),
    ([(0, 1)], "source, target, t"),
    ([(0, 1, "x")], "source, target, t"),
    ([(0, 1, 0.0)], r"\(0, 1\)"),
    ([(0, 1, 1.0)], r"\(0, 1\)"),
    ([(0, 1, -0.25)], r"\(0, 1\)"),
    ([(0, 1, 0.5), (1, 0, 1.5)], r"\(0, 1\)"),
    ([(0, 1, float("nan"))], r"\(0, 1\)"),
    ([(0, 1, float("inf"))], r"\(0, 1\)"),
    ([(0, 1, 1 - 1e-9)], r"\(0, 1\)"),    # rounds to 1.0 in the float32 the engine receives
    ([(0, 1, 1e-50)], r"\(0, 1\)"),       # ... to 0.0
    ([(0, 1, 1e300)], r"\(0, 1\)"),
])
def test_interpolate_at_rejects_bad_queries(model_r, queries, match):
    with pytest.raises(ValueError, match=match):
        model_r.interpolate_at(torch.rand(2, 3, 128, 128), queries)


@pytest.mark.parametrize("frames", [torch.rand(3, 128, 128), torch.rand(2, 4, 128, 128), torch.rand(0, 3, 128, 128), [1, 2]])
def test_interpolate_at_rejects_bad_frame_shapes(model_r, frames):
    with pytest.raises(ValueError, match="frames"):
        model_r.interpolate_at(frames, [(0, 0, 0.5)])


def test_interpolate_at_refuses_an_external_flow_backend():
    from gimmvfi_b200.model_f import GIMMVFI_F

    m = GIMMVFI_F()
    m.flow_backend = lambda a, b: None
    with pytest.raises(NotImplementedError, match="flow_backend"):
        m.interpolate_at(torch.rand(2, 3, 128, 128), [(0, 1, 0.5)])


# ------------------------------------------------------------------ C ABI
def test_query_entry_points_are_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "gimmvfi_b200.h")).read()
    names = ("gimmvfi_plan_queries", "gimmvfi_forward_queries", "gimmvfi_set_coord_range")
    for name in names:
        assert re.search(r"\bint %s\(" % name, header), name
    assert "typedef struct gimmvfi_queries" in header
    from gimmvfi_b200._lib import EXPORTS, default_lib

    lib = default_lib()
    for name in names:
        assert name in EXPORTS
        assert getattr(lib.dll, name) is not None


# ------------------------------------------------------------------ FrameRateConverter schedule (stub model, CPU padder)
class _Padder:
    """InputPadder on the host: (n,h,w,3) uint8 -> (n,3,h,w) float and back (the stub frames need no padding)"""

    def __init__(self, dims, divisor=32):
        self.ht, self.wd = dims[-2:]

    def pad_u8(self, f):
        return f.permute(0, 3, 1, 2).to(torch.float32) / 255.0

    def unpad_u8(self, pred, bgr=True):
        return (pred * 255.0).round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1)


class _StubModel:
    """interpolates by the weighted mean of the two frames; records every call as (frames, queries)"""

    def __init__(self):
        self.calls = []

    def _interpolate_at(self, frames, queries, ds, aux):
        assert aux is False
        self.calls.append((frames.clone(), list(queries)))
        return {"imgt_pred": torch.stack([(1 - t) * frames[a] + t * frames[b] for a, b, t in queries], 0)}


@pytest.fixture
def stub_video(monkeypatch):
    import gimmvfi_b200.video as V

    monkeypatch.setattr(V, "InputPadder", _Padder)
    return V


def _frame(j):
    """input frame j: channel c holds 10 j + c, so a frame's index can be read back and a BGR flip is visible"""
    f = torch.zeros(32, 64, 3, dtype=torch.uint8)
    for c in range(3):
        f[..., c] = 10 * j + c
    return f


RATES = [(24, 60), (60, 24), (25, 30), ("30000/1001", "60000/1001"), (Fraction(30), 30), ("29.97", 60), (30, 30)]


def _convert(V, fps_in, fps_out, n_frames, K):
    m = _StubModel()
    conv = V.FrameRateConverter(m, fps_in, fps_out, pairs_per_call=K)
    out = []
    for j in range(n_frames):
        got = conv.push(_frame(j))
        assert all(torch.is_tensor(g) for g in got)
        out += got
    out += conv.flush()
    assert conv.flush() == []
    return m, out


@pytest.mark.parametrize("K", [1, 3])
@pytest.mark.parametrize("fps_in,fps_out", RATES)
def test_frame_rate_converter_schedule(stub_video, fps_in, fps_out, K):
    n = 13
    m, out = _convert(stub_video, fps_in, fps_out, n, K)
    fi, fo = Fraction(str(fps_in)) if isinstance(fps_in, str) else Fraction(fps_in), Fraction(str(fps_out)) if isinstance(fps_out, str) else Fraction(fps_out)
    count = math.floor((n - 1) * fo / fi) + 1
    assert len(out) == count
    want_queries = []
    for k, o in enumerate(out):
        tau = k * fi / fo
        if tau.denominator == 1:   # the input frame itself, BGR-flipped, byte for byte
            assert torch.equal(o, _frame(int(tau)).flip(-1)), k
        else:
            a = math.floor(tau)
            t = float(np.float32(float(tau - a)))
            want_queries.append((a, a + 1, t))
            ref = ((1 - t) * (_frame(a).float() / 255) + t * (_frame(a + 1).float() / 255)) * 255
            assert (o.float() - ref.round()).abs().max() <= 1, k
    # the calls: every query once, in output order, with global frame indices read back from the frames' values
    sent = []
    for frames, qs in m.calls:
        idx = [int(round(f[0, 0, 0].item() * 255)) // 10 for f in frames]
        assert len(set(idx)) == len(idx) == frames.shape[0]                  # each frame at most once per call
        pairs = {(idx[a], idx[b]) for a, b, _ in qs}
        assert 1 <= len(pairs) <= K                                         # at most K pairs, each with queries
        assert sorted(idx) == sorted({i for p in pairs for i in p})         # exactly the frames of its pairs
        sent += [(idx[a], idx[b], t) for a, b, t in qs]
    assert sent == want_queries
    if fi == fo:
        assert m.calls == []
    # 60 -> 24 leaves pairs without any instant: they are never sent
    if (fi, fo) == (60, 24):
        assert len({(a, b) for a, b, _ in sent}) < n - 1


def test_frame_rate_converter_24_to_60_alternates(stub_video):
    m, out = _convert(stub_video, 24, 60, 5, 1)
    ts = [[round(t, 6) for _, _, t in qs] for _, qs in m.calls]
    assert ts == [[0.4, 0.8], [0.2, 0.6], [0.4, 0.8], [0.2, 0.6]]


@pytest.mark.parametrize("n", [1, 2])
def test_frame_rate_converter_short_clip(stub_video, n):
    """a clip shorter than one output period at 60 -> 24 gives its first frame only"""
    m, out = _convert(stub_video, 60, 24, n, 4)
    assert len(out) == 1 and torch.equal(out[0], _frame(0).flip(-1)) and m.calls == []


def test_frame_rate_converter_push_returns_what_is_complete(stub_video):
    m = _StubModel()
    conv = stub_video.FrameRateConverter(m, 24, 60, pairs_per_call=2)
    sizes = [len(conv.push(_frame(j))) for j in range(5)]
    # frame 0 at once; pairs (0,1), (1,2) in one call at frame 2 with the integral instant 2; pairs (2,3), (3,4) at frame 4
    assert sizes == [1, 0, 5, 0, 5] and len(m.calls) == 2
    assert conv.flush() == []


def _long_frame(j):
    """input frame j of a long clip: j in the first two channels"""
    f = torch.full((8, 8, 3), 7, dtype=torch.uint8)
    f[..., 0], f[..., 1] = j % 256, j // 256
    return f


# 30000/1001, 60000/1001 and 24000/1001 as the floats video readers report (and as a truncated decimal string): every 1001st instant
# falls a hair off an input frame instead of on it
NTSC = [(30000 / 1001, 60), (30000 / 1001, 24), ("29.97002997", 60), (60000 / 1001, 24), (24000 / 1001, 60), (60, 24000 / 1001)]
EXACT = {30000 / 1001: Fraction(30000, 1001), "29.97002997": Fraction(30000, 1001), 60000 / 1001: Fraction(60000, 1001),
         24000 / 1001: Fraction(24000, 1001), 60: Fraction(60), 24: Fraction(24)}


@pytest.mark.parametrize("fps_in,fps_out", NTSC)
def test_frame_rate_converter_inexact_rates_past_1001_outputs(stub_video, fps_in, fps_out):
    """more than 1001 outputs: every query sent has a float32 t strictly inside (0, 1), and the instants the exact rate puts on input
    frames come back as those frames, byte for byte"""
    m = _StubModel()
    conv = stub_video.FrameRateConverter(m, fps_in, fps_out, pairs_per_call=8)
    n = int(1400 * max(Fraction(1), conv.fps_in / conv.fps_out)) + 2
    out = []
    for j in range(n):
        out += conv.push(_long_frame(j))
    out += conv.flush()
    assert len(out) == math.floor((n - 1) * conv.fps_out / conv.fps_in) + 1 > 1001
    ts = [t for _, qs in m.calls for _, _, t in qs]
    assert ts and all(0.0 < float(np.float32(t)) < 1.0 and 1e-6 < t < 1 - 1e-6 for t in ts)
    step = EXACT[fps_in] / EXACT[fps_out]
    on_frame = [k for k in range(len(out)) if (k * step).denominator == 1]
    assert len(on_frame) >= 2 and on_frame[-1] >= 1001
    for k in on_frame:
        assert torch.equal(out[k], _long_frame(int(k * step)).flip(-1)), k


def test_frame_rate_converter_keeps_its_own_copy_of_the_last_frame(stub_video):
    """a caller that decodes into one reused buffer gets what it gets when it pushes a fresh tensor per frame"""
    _, ref = _convert(stub_video, 24, 60, 7, 3)
    conv = stub_video.FrameRateConverter(_StubModel(), 24, 60, pairs_per_call=3)
    buf, got = torch.zeros(32, 64, 3, dtype=torch.uint8), []
    for j in range(7):
        buf.copy_(_frame(j))
        got += conv.push(buf)
    got += conv.flush()
    assert len(got) == len(ref) and all(torch.equal(a, b) for a, b in zip(got, ref))


@pytest.mark.parametrize("bad", [0, -24, "0/1", "abc", None, True])
def test_frame_rate_converter_refuses_bad_rates(bad):
    from gimmvfi_b200.video import FrameRateConverter

    with pytest.raises(ValueError):
        FrameRateConverter(_StubModel(), bad, 30)
    with pytest.raises(ValueError):
        FrameRateConverter(_StubModel(), 30, 60, pairs_per_call=0)


# ------------------------------------------------------------------ host simulation: a query list against per-pair forwards
@pytest.fixture(scope="module")
def sim(weights0):
    sys.path.insert(0, os.path.join(HERE, "hostsim"))
    from harness import hostsim_engine

    e = hostsim_engine()
    e.load_state_dict(weights0)
    return e


# (0,1) has 3 timesteps (GIMM's pyramid lookup), (2,2) a self pair with 2 and the reversed (1,0) and (4,2) 1 each (volume-free lookup);
# frame 3 is unused, and the queries of one pair are interleaved with the others'
QUERIES = [(0, 1, 0.2), (2, 2, 0.3), (1, 0, 0.6), (0, 1, 0.5), (4, 2, 0.25), (2, 2, 0.7), (0, 1, 0.8)]


def test_hostsim_queries_match_per_pair_forwards(sim):
    """The simulation runs precision mode 0, whose GIMM correlation always takes the pyramid: the volume-free lookup of the pairs with at
    most 2 timesteps needs a tensor-core mode, and tests/test_queries_gpu.py covers the mixed paths in one call.  Outputs upstream
    of the splat are bit-identical to forward() with B = 1 at the pair's own timestep list; the splat sums in a thread-dependent order,
    so the outputs after it may differ in the last bits."""
    torch.set_grad_enabled(False)
    from gimmvfi_r_oracle import sample_coord_input

    H, W = 128, 128
    fr = synth_batch(3, H, W, seed=23)
    frames = fr.permute(0, 2, 1, 3, 4).reshape(-1, 3, H, W)[:5].contiguous()
    try:
        sim.set_debug(True)
        q = sim.forward_queries(frames, QUERIES, None)
        grid = sim.tap("query.coords")                    # the last slot: (0,1) at 0.8
        assert torch.equal(grid, sample_coord_input(1, (H, W), [0.8], 1.0).reshape(1, H, W, 3))
        sim.set_debug(False)
        pairs, index = sim.query_pairs(QUERIES)
        assert pairs == [(0, 1), (2, 2), (1, 0), (4, 2)] and index == [0, 1, 2, 0, 3, 1, 0]
        assert q["imgt_pred"].shape == (7, 3, H, W) and q["raft_flow"].shape == (4, 2, 2, H, W) and q["ninrflow"].shape == (7, 2, 1, H, W)
        for p, (a, b) in enumerate(pairs):
            mine = [i for i, x in enumerate(index) if x == p]
            ts = [QUERIES[i][2] for i in mine]
            T = len(ts)
            coords = torch.stack([sample_coord_input(1, (H, W), [t], 1.0) for t in ts], 0).contiguous()
            tt = torch.tensor(ts).unsqueeze(1).contiguous()
            xs = torch.stack([frames[a], frames[b]], 1).unsqueeze(0).contiguous()
            one = sim.forward(xs, coords, tt, None)
            assert torch.equal(q["raft_flow"][p:p + 1], one["raft_flow"]), (a, b)
            assert torch.equal(q["nflow"][p:p + 1], one["nflow"]), (a, b)
            for k, bar in (("imgt_pred", 1e-5), ("ninrflow", 1e-5), ("img_warp_4", 1e-5), ("flowt", 1e-4), ("flowt0_1", 1e-4)):
                for i, qi in enumerate(mine):
                    assert (q[k][qi] - one[k][i, 0]).abs().max() <= bar, (k, a, b, i)
            assert T == (3 if (a, b) == (0, 1) else 2 if (a, b) == (2, 2) else 1)
    finally:
        sim.set_debug(False)


@pytest.mark.parametrize("t", [0.0, 1.0, float("nan"), -0.5])
def test_hostsim_queries_refuse_t_outside_the_open_interval(sim, t):
    from gimmvfi_b200._lib import GimmvfiError

    with pytest.raises(GimmvfiError, match="strictly inside"):
        sim.forward_queries(torch.rand(2, 3, 128, 128), [(0, 1, 0.5), (0, 1, t)], None)


def test_hostsim_query_plans_depend_on_structure_only(sim):
    """two query lists with the same pairs and counts but other t share one cached plan; another count makes a new one"""
    sim._plans.clear()
    a = sim.queries_workspace_bytes(3, [(0, 1, 0.25), (1, 2, 0.5), (0, 1, 0.75)], 128, 128, None, 128, 128)
    b = sim.queries_workspace_bytes(3, [(0, 1, 0.1), (1, 2, 0.9), (0, 1, 0.3)], 128, 128, None, 128, 128)
    assert a == b and len([k for k in sim._plans if k[0] == "queries"]) == 1
    sim.queries_workspace_bytes(3, [(0, 1, 0.25), (1, 2, 0.5), (1, 2, 0.75)], 128, 128, None, 128, 128)
    assert len([k for k in sim._plans if k[0] == "queries"]) == 2
