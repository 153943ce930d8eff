"""Scene-cut detection on the GPU: gimmvfi_op_scene_sums against cv2's RGB -> HSV (every 8-bit colour; random frames up to 2160x3840,
odd sizes, aligned and unaligned stacks), bitwise-equal reruns, scene_scores' refusals, and a clip of two shots through FrameRateConverter
and VideoInterpolator on GIMM-VFI-R and -F with the threshold at 27: exactly the one cut, no engine work for it, the nearer input frame in
its place, and every other output within 1 uint8 level of the same object run without a threshold (the splat's float-atomic noise)."""
import numpy as np
import pytest
import torch

from gimmvfi_b200 import GIMMVFI_R
from gimmvfi_b200.model_f import GIMMVFI_F
from gimmvfi_b200.synth import synth_batch
from gimmvfi_b200.weights import random_state_dict, random_state_dict_f

pytestmark = pytest.mark.gpu
DEV = "cuda"


def cv2_sums(a, b):
    cv2 = pytest.importorskip("cv2")
    hsv = lambda x: cv2.cvtColor(np.ascontiguousarray(x), cv2.COLOR_RGB2HSV).astype(np.int64)
    return np.stack([np.abs(hsv(x) - hsv(y)).reshape(-1, 3).sum(0) for x, y in zip(a, b)], 0)


def test_every_colour_against_cv2():
    """2^24 pairs of 1x1 frames: every RGB colour against black (HSV (0, 0, 0)) -> the colour's H + S + V"""
    cv2 = pytest.importorskip("cv2")
    from gimmvfi_b200.video import _scene_sums

    c = torch.arange(1 << 24, dtype=torch.int64, device=DEV)
    a = torch.stack([(c >> 16) & 255, (c >> 8) & 255, c & 255], -1).to(torch.uint8).reshape(-1, 1, 1, 3).contiguous()
    got = _scene_sums(a, torch.zeros_like(a)).cpu().numpy()
    want = cv2.cvtColor(a.cpu().numpy().reshape(4096, 4096, 3), cv2.COLOR_RGB2HSV).reshape(-1, 3).astype(np.int64)
    assert np.array_equal(got, want), np.argwhere(got != want)[:5]


def _unaligned(frames):
    """the same frames in a stack that starts one byte past an allocation (no 16-byte loads)"""
    buf = torch.empty(frames.numel() + 16, dtype=torch.uint8, device=DEV)
    v = buf[1:1 + frames.numel()].view(frames.shape)
    v.copy_(frames)
    return v


@pytest.mark.parametrize("size", [(1, 1), (5, 5), (8, 8), (9, 8), (17, 31), (120, 150), (1080, 1920), (1079, 1917), (2160, 3840),
                                  (2159, 3839)])
def test_sums_and_scores_against_cv2(size):
    from gimmvfi_b200.video import _scene_sums, scene_scores

    h, w = size
    rng = np.random.default_rng(h * 7919 + w)
    host = rng.integers(0, 256, (6, h, w, 3), dtype=np.uint8)
    host[3] = host[2] // 2 + 40
    want = cv2_sums(host[:-1], host[1:])
    frames = torch.from_numpy(host).to(DEV)
    for stack in (frames, _unaligned(frames)):
        for n in (1, 5):
            got = _scene_sums(stack[:n], stack[1:n + 1]).cpu().numpy()
            assert np.array_equal(got, want[:n]), (size, n)
    scores = scene_scores(frames)
    assert scores.dtype == torch.float64 and scores.device.type == "cpu"
    assert np.array_equal(scores.numpy(), want.sum(1).astype(np.float64) / (3 * h * w))


@pytest.mark.parametrize("size", [(2160, 3840), (1079, 1917), (4, 4)])
def test_two_runs_are_bitwise_equal(size):
    from gimmvfi_b200.video import _scene_sums

    g = torch.Generator(device=DEV).manual_seed(size[0])
    frames = torch.randint(0, 256, (17, *size, 3), dtype=torch.uint8, device=DEV, generator=g)
    r1 = _scene_sums(frames[:-1], frames[1:]).cpu()
    r2 = _scene_sums(frames[:-1], frames[1:]).cpu()
    assert torch.equal(r1, r2)


def test_scene_scores_refuses_bad_input():
    from gimmvfi_b200.video import scene_scores

    good = torch.zeros(3, 8, 8, 3, dtype=torch.uint8, device=DEV)
    for bad, match in ((good.cpu(), "CUDA"), (good.float(), "uint8"), (good[:1], "2 frames"), (good[:, :, ::2], "contiguous"),
                       (torch.zeros(3, 8, 8, 4, dtype=torch.uint8, device=DEV), "uint8")):
        with pytest.raises(ValueError, match=match):
            scene_scores(bad)


# ------------------------------------------------------------------ a clip of two shots through the video classes
def make_model(kind):
    if kind == "R":
        m = GIMMVFI_R(None, seed=0).to(DEV).eval()
        m.load_state_dict(random_state_dict(0), strict=True)
    else:
        m = GIMMVFI_F(None).to(DEV).eval()
        m.load_state_dict(random_state_dict_f(0), strict=True)
    m.kind = kind
    m.tensor_cores = 4
    return m


@pytest.fixture(scope="module", params=["R", "F"])
def model(request):
    yield make_model(request.param)


CUT = 5   # input frame 5 starts the second shot


def two_shots(kind):
    """10 uint8 (h,w,3) frames: 5 of a synth_batch frame of seed 3, then 5 of seed 5, each shifted by one pixel diagonally per frame.
    Measured with cv2: within a shot 21.5-21.7 then 16.9-17.0 at 120x150, 20.2-20.3 then 16.5-16.6 at 128x160; the cut 43.2 and 42.3."""
    H, W = (128, 160) if kind == "F" else (120, 150)
    out = []
    for seed in (3, 5):
        src = synth_batch(1, H + CUT, W + CUT, seed=seed)[0, :, 0]
        out += [(src[:, i:i + H, i:i + W].permute(1, 2, 0) * 255).to(torch.uint8).contiguous().to(DEV) for i in range(CUT)]
    return out


def test_two_shot_scores():
    from gimmvfi_b200.video import scene_scores

    for kind in ("R", "F"):
        s = scene_scores(torch.stack(two_shots(kind), 0)).tolist()
        assert all(x < 27 for i, x in enumerate(s) if i != CUT - 1) and s[CUT - 1] >= 27, (kind, s)
        print(kind, "scores", ["%.2f" % x for x in s])


class Recorder:
    """wraps one of the model's entry points and records the (source, target) input frames of every pair it is sent"""

    def __init__(self, model, name, padded):
        self.model, self.name, self.pairs, self.calls = model, name, [], 0
        idx = lambda f: next(i for i, p in enumerate(padded) if torch.equal(p, f))
        orig = getattr(model, name)

        def rec(*a, **k):
            self.calls += 1
            if name == "_interpolate_at":
                self.pairs += sorted({(idx(a[0][s]), idx(a[0][t])) for s, t, _ in a[1]})
            elif name == "_interpolate_clip":
                self.pairs += [(idx(a[0][s]), idx(a[0][t])) for s, t in a[1]]
            else:
                self.pairs.append((idx(a[0][0, :, 0]), idx(a[0][0, :, 1])))
            return orig(*a, **k)

        setattr(model, name, rec)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        delattr(self.model, self.name)


def _padded(u8):
    from gimmvfi_b200.video import InputPadder

    return list(InputPadder(u8[0].shape[:2], 32).pad_u8(torch.stack(u8, 0)).unbind(0))


@pytest.mark.parametrize("K", [1, 4])
def test_converter_two_shots(model, K):
    from gimmvfi_b200.video import FrameRateConverter

    u8 = two_shots(model.kind)
    res = {}
    for thr in (None, 27):
        conv = FrameRateConverter(model, 24, 60, pairs_per_call=K, scene_threshold=thr)
        with Recorder(model, "_interpolate_at", _padded(u8)) as rec:
            out = []
            for f in u8:
                out += conv.push(f)
            out += conv.flush()
        res[thr] = (out, rec.pairs, conv.cuts)
    (ref, ref_pairs, ref_cuts), (got, pairs, cuts) = res[None], res[27]
    assert ref_cuts == [] and cuts == [CUT]
    assert sorted(ref_pairs) == [(j - 1, j) for j in range(1, 10)]
    assert sorted(pairs) == [(j - 1, j) for j in range(1, 10) if j != CUT]
    assert len(got) == len(ref) == 9 * 60 // 24 + 1
    for k, (x, y) in enumerate(zip(got, ref)):
        tau = k * 24 / 60
        if CUT - 1 < tau < CUT:
            near = u8[CUT - 1] if tau - (CUT - 1) <= 0.5 else u8[CUT]
            assert torch.equal(x, near.flip(-1)), k
        else:
            assert x.shape == y.shape and (x.int() - y.int()).abs().max().item() <= 1, k


@pytest.mark.parametrize("with_flow", [False, True])
@pytest.mark.parametrize("K", [1, 3])
def test_interpolator_two_shots(model, K, with_flow):
    from gimmvfi_b200.video import VideoInterpolator

    N = 4
    u8 = two_shots(model.kind)
    res = {}
    for thr in (None, 27):
        vi = VideoInterpolator(model, N=N, with_flow=with_flow, pairs_per_call=K, scene_threshold=thr)
        with Recorder(model, "_interpolate" if K == 1 else "_interpolate_clip", _padded(u8)) as rec:
            frames, flows = [], []
            for f in u8 + [None]:
                got = vi.push(f) if f is not None else vi.flush()
                a, b = got if with_flow else (got, [])
                frames += a
                flows += b
        res[thr] = (frames, flows, rec.pairs, vi.cuts)
    (ref, ref_fl, ref_pairs, ref_cuts), (got, fl, pairs, cuts) = res[None], res[27]
    assert ref_cuts == [] and cuts == [CUT]
    assert ref_pairs == [(j - 1, j) for j in range(1, 10)]
    assert pairs == [(j - 1, j) for j in range(1, 10) if j != CUT]
    assert len(got) == len(ref) == 9 * (N - 1) and len(fl) == len(ref_fl) == (9 * (N - 1) if with_flow else 0)
    cut = [p * (N - 1) + i - 1 for p in range(9) for i in range(1, N) if p + 1 == CUT]
    for k in range(len(got)):
        if k in cut:
            i = k % (N - 1) + 1
            assert torch.equal(got[k], (u8[CUT - 1] if 2 * i <= N else u8[CUT]).flip(-1)), k
        else:
            assert (got[k].int() - ref[k].int()).abs().max().item() <= 1, k
    for k in range(len(fl)):
        assert fl[k].shape == ref_fl[k].shape, k
        if k in cut:   # the colour wheel of a zero flow is white
            assert bool((fl[k] == 255).all()), k
        else:
            # flow_to_image's wheel has a seam at angle pi (colour 54 is (255, 0, 43), colour 0 is (255, 0, 0)): where a flow points
            # along +x, the splat's float-atomic noise can flip the sign of v and move the blue channel by up to 43 levels
            d = (fl[k].int() - ref_fl[k].int()).abs().amax(-1)
            assert d.max().item() <= 43 and (d > 1).float().mean().item() <= 0.01, (k, d.max().item(), (d > 1).sum().item())
