"""The clip form of GIMM-VFI-R / -F without a GPU: interpolate's argument checks, VideoInterpolator's buffering with a stub model, the
C exports, and the host simulation of the engine running a clip against per-pair forwards."""
import os
import re
import sys

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


@pytest.mark.parametrize("pairs,match", [
    ([], "empty"),
    ([(0, 3)], "outside"),
    ([(-1, 0)], "outside"),
    ([(0, 1), (2, 1)], "outside"),
    ([(0,)], "source, target"),
])
def test_interpolate_rejects_bad_pairs(model_r, pairs, match):
    frames = torch.rand(2, 3, 128, 128)
    with pytest.raises(ValueError, match=match):
        model_r.interpolate(frames, pairs, [0.5])


@pytest.mark.parametrize("frames", [torch.rand(3, 128, 128), torch.rand(2, 4, 128, 128), torch.rand(0, 3, 128, 128)])
def test_interpolate_rejects_bad_frame_shapes(model_r, frames):
    with pytest.raises(ValueError, match="frames"):
        model_r.interpolate(frames, [(0, 0)], [0.5])


@pytest.mark.parametrize("t", [[], 0.5, None, ["a"]])
def test_interpolate_rejects_bad_timesteps(model_r, t):
    with pytest.raises(ValueError, match="t must"):
        model_r.interpolate(torch.rand(2, 3, 128, 128), [(0, 1)], t)


def test_interpolate_refuses_an_external_flow_backend():
    from gimmvfi_b200.model_f import GIMMVFI_F

    m = GIMMVFI_F()
    m.flow_backend = lambda a, b: None
    with pytest.raises(NotImplementedError, match="flow_backend"):
        m.interpolate(torch.rand(2, 3, 128, 128), [(0, 1)], [0.5])


# ------------------------------------------------------------------ C ABI
def test_clip_entry_points_are_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "gimmvfi_b200.h")).read()
    for name in ("gimmvfi_plan_clip", "gimmvfi_forward_clip"):
        assert re.search(r"\bint %s\(" % name, header), name
    assert "typedef struct gimmvfi_clip" in header
    from gimmvfi_b200._lib import EXPORTS, default_lib

    lib = default_lib()
    for name in ("gimmvfi_plan_clip", "gimmvfi_forward_clip"):
        assert name in EXPORTS
        assert getattr(lib.dll, name) is not None


# ------------------------------------------------------------------ VideoInterpolator buffering (stub model, CPU padder)
class _Padder:
    """InputPadder on the host: (n,h,w,3) uint8 -> (n,3,h,w) float and back (no padding: the stub frames are multiples of 32)"""

    def __init__(self, dims, divisor=32):
        self.ht, self.wd = dims[-2:]

    def pad_u8(self, f):
        return f.permute(0, 3, 1, 2).to(torch.float32) / 255.0

    def unpad_u8(self, pred, bgr=True):
        return (pred * 255.0).round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1)

    def unpad_box(self, ht, wd):
        return 0, ht, 0, wd


class _StubModel:
    """interpolates by a weighted mean (its value says which pair and timestep made it); records every call"""

    def __init__(self):
        self.clip_calls, self.pair_calls = [], 0

    def _interpolate_clip(self, frames, pairs, t, ds, aux):
        self.clip_calls.append((frames.shape[0], list(pairs), list(t), aux))
        ims = [torch.stack([(1 - ti) * frames[a] + ti * frames[b] for a, b in pairs], 0) for ti in t]
        out = {"imgt_pred": ims}
        if aux:
            fl = [torch.stack([torch.full((2,) + frames.shape[-2:], float(p * 10 + i)) for p in range(len(pairs))], 0)
                  for i in range(len(t))]
            out["flowt"] = [f.squeeze() for f in fl]
        return out


@pytest.fixture
def stub_video(monkeypatch):
    import gimmvfi_b200.video as V

    monkeypatch.setattr(V, "InputPadder", _Padder)
    monkeypatch.setattr(V, "flow_images", lambda padder, flowt, bgr: [f[0, 0, 0].item() for f in flowt])
    return V


def _frame(v):
    return torch.full((32, 64, 3), v, dtype=torch.uint8)


@pytest.mark.parametrize("K", [2, 3, 4])
def test_video_interpolator_buffers_pairs_in_clip_order(stub_video, K):
    m = _StubModel()
    N, n_frames = 4, 9
    vi = stub_video.VideoInterpolator(m, N=N, pairs_per_call=K)
    vals = [8 * j for j in range(n_frames)]   # (every interpolated value an integer: no rounding ties)
    got = []
    for j, v in enumerate(vals):
        out = vi.push(_frame(v))
        # output only when K pairs are waiting
        assert (len(out) > 0) == (j > 0 and j % K == 0)
        got += out
    got += vi.flush()
    assert vi.flush() == []
    # N-1 frames per pair, pairs in clip order, timesteps in order within a pair
    want = [round(vals[p] + (i / N) * (vals[p + 1] - vals[p])) for p in range(n_frames - 1) for i in range(1, N)]
    assert [int(f[0, 0, 0]) for f in got] == want
    # each call takes K pairs of consecutive frames (the rest at flush), each frame once
    sizes = [c[0] - 1 for c in m.clip_calls]
    assert sizes == [K] * ((n_frames - 1) // K) + ([(n_frames - 1) % K] if (n_frames - 1) % K else [])
    for c in m.clip_calls:
        assert c[1] == [(i, i + 1) for i in range(c[0] - 1)] and c[2] == [i / N for i in range(1, N)] and c[3] is False


def test_video_interpolator_buffered_flow_pictures(stub_video):
    m = _StubModel()
    vi = stub_video.VideoInterpolator(m, N=3, pairs_per_call=2, with_flow=True)
    frames, flows = [], []
    for v in (0, 30, 60, 90):
        f, fl = vi.push(_frame(v))
        frames += f
        flows += fl
    f, fl = vi.flush()
    frames += f
    flows += fl
    assert len(frames) == len(flows) == 3 * 2
    # pair p, timestep i -> the stub's flow value p*10 + i, pair by pair (pair numbers restart in each call)
    assert flows == [0.0, 1.0, 10.0, 11.0, 0.0, 1.0]
    assert all(c[3] == ("flowt",) for c in m.clip_calls)


def test_video_interpolator_refuses_bad_pairs_per_call():
    from gimmvfi_b200.video import VideoInterpolator

    with pytest.raises(ValueError):
        VideoInterpolator(_StubModel(), N=2, pairs_per_call=0)


@pytest.mark.parametrize("N", [1, 0])
def test_video_interpolator_refuses_n_below_2(N):
    """N = 1 would schedule no frame between two inputs"""
    from gimmvfi_b200.video import VideoInterpolator

    with pytest.raises(ValueError, match="N must be >= 2"):
        VideoInterpolator(_StubModel(), N=N)


def test_video_interpolator_frame_size_change_needs_flush(stub_video):
    vi = stub_video.VideoInterpolator(_StubModel(), N=2, pairs_per_call=3)
    vi.push(_frame(0))
    vi.push(_frame(10))
    with pytest.raises(ValueError, match="flush"):
        vi.push(torch.zeros(64, 64, 3, dtype=torch.uint8))


# ------------------------------------------------------------------ host simulation: a clip against per-pair forwards
@pytest.fixture(scope="module")
def sim(weights0):
    sys.path.insert(0, os.path.join(HERE, "hostsim"))
    from harness import hostsim_engine

    e = hostsim_engine()
    e.load_state_dict(weights0)
    return e


def test_hostsim_clip_matches_per_pair_forwards(sim):
    """3 frames; a consecutive, a reversed and a self pair.  Outputs upstream of the splat are bit-identical; the
    splat sums in a thread-dependent order, so the outputs after it may differ in the last bits."""
    torch.set_grad_enabled(False)
    H, W, ts = 128, 128, [0.25]
    fr = synth_batch(2, H, W, seed=21)
    frames = torch.stack([fr[0, :, 0], fr[0, :, 1], fr[1, :, 1]], 0).contiguous()
    pairs = [(0, 1), (2, 1), (1, 1)]
    from gimmvfi_r_oracle import sample_coord_input

    P, T = len(pairs), len(ts)
    coords = torch.stack([sample_coord_input(P, (H, W), [t], 1.0) for t in ts], 0).contiguous()
    tt = torch.tensor(ts).unsqueeze(1).expand(T, P).contiguous()
    clip = sim.forward_clip(frames, pairs, coords, tt, None)
    assert sim.clip_workspace_bytes(3, pairs, H, W, T, None, H, W) > 0
    for p, (a, b) in enumerate(pairs):
        xs = torch.stack([frames[a], frames[b]], 1).unsqueeze(0).contiguous()
        one = sim.forward(xs, coords[:, p:p + 1].contiguous(), tt[:, p:p + 1].contiguous(), None)
        assert torch.equal(clip["raft_flow"][p:p + 1], one["raft_flow"])
        assert torch.equal(clip["nflow"][p:p + 1], one["nflow"])
        for k, bar in (("imgt_pred", 1e-5), ("ninrflow", 1e-5), ("img_warp_4", 1e-5), ("flowt", 1e-4), ("flowt0_1", 1e-4)):   # (flows in px)
            assert (clip[k][:, p:p + 1] - one[k]).abs().max() <= bar, k


def test_clip_plan_cache_is_bounded(sim):
    """a plan per pair list, but only the most recent EngineHandle.CLIP_PLANS lists stay cached"""
    sizes = set()
    for k in range(sim.CLIP_PLANS + 4):
        pairs = [(0, 1)] * (k + 1)
        sizes.add(sim.clip_workspace_bytes(2, pairs, 128, 128, 1, None, 128, 128))
    assert len(sizes) > 1   # (the volumes grow with the pairs)
    clip_keys = [key for key in sim._plans if key[0] == "clip"]
    assert len(clip_keys) == sim.CLIP_PLANS
    assert clip_keys[-1][2] == tuple([(0, 1)] * (sim.CLIP_PLANS + 4))   # the most recent list is kept
