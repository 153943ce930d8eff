"""Shutter-angle motion blur on the GPU: gimmvfi_op_blend_u8 bit-identical to its host simulation from 1x1 up to 2160x3840 with 16-byte and
byte-wise uint8 loads and stores, reruns bitwise equal; FrameRateConverter(shutter_angle=...) through GIMM-VFI-R and -F (seeded weights,
precision mode 4) within 1 uint8 level of a float64 blend of interpolate_at on the same queries over the same kept samples (the splat's
float atomics move a sub-frame by a level), S = 1 within 1 level of the converter without a shutter, and a clip of two shots through R:
no query for the cut pair, and no output mixing the shots."""
import ctypes as C
import math
import os
import sys
from fractions import Fraction

import numpy as np
import pytest
import torch

from gimmvfi_b200 import GIMMVFI_R
from gimmvfi_b200.model_f import GIMMVFI_F
from gimmvfi_b200.synth import synth_batch
from gimmvfi_b200.weights import random_state_dict, random_state_dict_f

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
SNAP = Fraction(1, 10 ** 6)


@pytest.fixture(scope="module")
def simlib():
    sys.path.insert(0, os.path.join(HERE, "hostsim"))
    import harness

    from gimmvfi_b200._lib import Lib

    return Lib(harness.build_hostsim())


def _offset(x, k):
    """a copy of x in a buffer that starts k bytes past an allocation"""
    buf = torch.empty(x.numel() * x.element_size() + 64, dtype=torch.uint8, device=x.device)
    v = buf[k:k + x.numel() * x.element_size()].view(x.dtype).view(x.shape)
    v.copy_(x)
    return v


def sim_blend(lib, sources, H, W, top, left, h, w, bgr):
    srcs = [s.cpu().numpy() for s in sources]
    dst = np.empty((h, w, 3), np.uint8)
    n = len(srcs)
    ptrs = (C.c_void_p * n)(*[s.ctypes.data for s in srcs])
    kinds = (C.c_int * n)(*[int(s.dtype == np.float32) for s in srcs])
    lib.check(lib.dll.gimmvfi_op_blend_u8(ptrs, kinds, n, H, W, top, left, C.c_void_p(dst.ctypes.data), h, w, int(bgr), None))
    return torch.from_numpy(dst)


def blend_into(sources, p, bgr, dst):
    """gimmvfi_op_blend_u8 through the C ABI into a given (h,w,3) uint8 dst (blend_u8 allocates its own, always 16-byte aligned)"""
    from gimmvfi_b200._lib import default_lib

    H, W = p.padded_shape
    top, _, left, _ = p.unpad_box(H, W)
    n = len(sources)
    lib = default_lib()
    ptrs = (C.c_void_p * n)(*[s.data_ptr() for s in sources])
    kinds = (C.c_int * n)(*[int(s.dtype == torch.float32) for s in sources])
    lib.check(lib.dll.gimmvfi_op_blend_u8(ptrs, kinds, n, H, W, top, left, C.c_void_p(dst.data_ptr()), p.ht, p.wd, int(bgr),
                                          C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    return dst


@pytest.mark.parametrize("size", [(1, 1), (5, 7), (30, 50), (128, 160), (1079, 1917), (1080, 1920), (2160, 3840)])
def test_op_matches_host_simulation(simlib, size):
    from gimmvfi_b200.video import InputPadder, blend_u8

    h, w = size
    p = InputPadder(size, 32)
    H, W = p.padded_shape
    top, _, left, _ = p.unpad_box(H, W)
    g = torch.Generator(device=DEV).manual_seed(h * 7 + w)
    n = 7 if h * w > 1 << 20 else 13
    srcs = [torch.rand(3, H, W, device=DEV, generator=g) * 1.2 - 0.1 if i % 3 != 1 else
            torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, device=DEV, generator=g) for i in range(n)]
    for bgr in (True, False):
        want = sim_blend(simlib, srcs, H, W, top, left, h, w, bgr)
        got = blend_u8(srcs, p, bgr)
        assert torch.equal(got.cpu(), want), (size, bgr)
        # uint8 sources one byte off a 16-byte boundary: the byte-wise loads
        odd = [s if s.dtype == torch.float32 else _offset(s, 1) for s in srcs]
        assert torch.equal(blend_u8(odd, p, bgr).cpu(), want), (size, bgr)
        # an output one byte off a 16-byte boundary: the byte-wise stores
        dst = _offset(torch.zeros(h, w, 3, dtype=torch.uint8, device=DEV), 1)
        assert dst.data_ptr() % 16 == 1
        assert torch.equal(blend_into(odd, p, bgr, dst).cpu(), want), (size, bgr)
        assert torch.equal(blend_u8(srcs, p, bgr), got)   # reruns are bitwise equal
    # 63 sources, a 16-byte aligned frame among them and copies of one frame
    u = srcs[1]
    assert torch.equal(blend_u8([u] * 63, p, False), u)


def test_op_refuses_bad_sources():
    from gimmvfi_b200.video import InputPadder, blend_u8

    p = InputPadder((30, 50), 32)
    u = torch.zeros(30, 50, 3, dtype=torch.uint8, device=DEV)
    for bad in ([], [u] * 64, [u[:, :-1]], [u.float()], [torch.zeros(3, 30, 50, device=DEV)], [u.transpose(0, 1)]):
        with pytest.raises(ValueError, match="blend_u8"):
            blend_u8(bad, p)


# ------------------------------------------------------------------ through the models
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


def clip(n, h, w, seed=1):
    """n frames of a smooth pattern moving a few pixels per frame"""
    g = torch.Generator(device="cpu").manual_seed(seed)
    base = torch.rand(3, h // 16 + 4, w // 16 + 4, generator=g)
    big = torch.nn.functional.interpolate(base[None], size=(h + 4 * n, w + 4 * n), mode="bicubic", align_corners=False)[0].clamp(0, 1)
    return [(big[:, 3 * j:3 * j + h, 2 * j:2 * j + w].permute(1, 2, 0) * 255).to(torch.uint8).contiguous().to(DEV) for j in range(n)]


def kept_samples(fps_in, fps_out, n, A, S, cuts=()):
    """each output's kept samples, ("frame", f) or ("query", a, a + 1, t), as the converter documents them"""
    step = Fraction(fps_in) / Fraction(fps_out)
    wnd = Fraction(A) / 360 * step
    shot = lambda f: sum(1 for c in cuts if c <= f)
    outs, k = [], 0
    while k * step <= n - 1:
        tau, samples = k * step, []
        for i in range(S):
            x = tau - wnd / 2 + Fraction(2 * i + 1, 2 * S) * wnd
            if x < 0 or x > n - 1:
                continue
            a, off = math.floor(x), x - math.floor(x)
            src = (("frame", a) if off <= SNAP else ("frame", a + 1) if off >= 1 - SNAP else
                   ("frame", a if off <= Fraction(1, 2) else a + 1) if a + 1 in cuts else ("query", a, a + 1, float(np.float32(float(off)))))
            samples.append((x == tau, src))
        own = shot(next(s for m, s in samples if m)[1])
        outs.append([s for _, s in samples if shot(s[1]) == own])
        k += 1
    return outs


def run(model, u8, fps_in, fps_out, K, A=None, S=7, threshold=None):
    """the converter's outputs, and each engine call's queries as (input a, input b, t)"""
    from gimmvfi_b200.video import FrameRateConverter, InputPadder

    padded = list(InputPadder(u8[0].shape[:2], 32).pad_u8(torch.stack(u8, 0)).unbind(0))
    idx = lambda f: next(i for i, p in enumerate(padded) if torch.equal(p, f))
    calls, orig = [], model._interpolate_at

    def rec(frames, queries, ds, aux):
        calls.append([(idx(frames[a]), idx(frames[b]), t) for a, b, t in queries])
        return orig(frames, queries, ds, aux)

    model._interpolate_at = rec
    try:
        conv = FrameRateConverter(model, fps_in, fps_out, pairs_per_call=K, shutter_angle=A, shutter_samples=S, scene_threshold=threshold)
        out = []
        for f in u8:
            out += conv.push(f)
        out += conv.flush()
    finally:
        del model._interpolate_at
    return out, calls, padded, conv


def reference(model, u8, padded, calls, kept):
    """interpolate_at on each recorded call's queries, blended in float64 over the kept samples -> uint8 BGR"""
    from gimmvfi_b200.video import InputPadder

    p = InputPadder(u8[0].shape[:2], 32)
    h, w = p.ht, p.wd
    top, _, left, _ = p.unpad_box(*p.padded_shape)
    sub = {}
    for qs in calls:
        used = sorted({f for a, b, _ in qs for f in (a, b)})
        local = {f: i for i, f in enumerate(used)}
        got = model.interpolate_at(torch.stack([padded[f] for f in used], 0), [(local[a], local[b], t) for a, b, t in qs])["imgt_pred"]
        for q, x in zip(qs, got):
            sub[q] = x[:, top:top + h, left:left + w].permute(1, 2, 0).double() * 255
    out = []
    for samples in kept:
        acc = sum(u8[s[1]].double() if s[0] == "frame" else sub[s[1:]] for s in samples) / len(samples)
        out.append(acc.clamp(0, 255).to(torch.uint8).flip(-1))
    return out


def _close(a, b):
    return a.shape == b.shape and (a.int() - b.int()).abs().max().item() <= 1


@pytest.mark.parametrize("K", [1, 2])
def test_models_against_float64_blend(model, K):
    u8 = clip(9, 128, 160)
    out, calls, padded, _ = run(model, u8, 60, 24, K, A=180, S=5)
    kept = kept_samples(60, 24, 9, 180, 5)
    assert len(out) == len(kept) and any(len(s) > 1 for s in kept)
    ref = reference(model, u8, padded, calls, kept)
    for k, (o, r) in enumerate(zip(out, ref)):
        assert _close(o, r), (model.kind, K, k, (o.int() - r.int()).abs().max().item())
    # S = 1 against the converter without a shutter; frames passed through are exact
    plain, _, _, _ = run(model, u8, 60, 24, K)
    one, _, _, _ = run(model, u8, 60, 24, K, A=180, S=1)
    assert len(one) == len(plain)
    for k, (a, b) in enumerate(zip(one, plain)):
        assert _close(a, b), k
        if (k * Fraction(60, 24)).denominator == 1:
            assert torch.equal(a, u8[k * 60 // 24].flip(-1)) and torch.equal(b, a), k


def test_r_1080p():
    m = make_model("R")
    u8 = clip(4, 1088, 1920)
    out, calls, padded, _ = run(m, u8, 60, 24, 1, A=180, S=5)
    kept = kept_samples(60, 24, 4, 180, 5)
    ref = reference(m, u8, padded, calls, kept)
    assert len(out) == len(kept) == 2
    for k, (o, r) in enumerate(zip(out, ref)):
        assert _close(o, r), (k, (o.int() - r.int()).abs().max().item())


CUT = 5


def two_shots(H=120, W=150):
    """10 frames: 5 of a synth_batch frame of seed 3, then 5 of seed 5, each shifted by one pixel diagonally per frame (the cut scores
    about 43, frames within a shot below 22)"""
    out = []
    for seed in (3, 5):
        src = synth_batch(1, H + CUT, W + CUT, seed=seed)[0, :, 0]
        out += [(src[:, i:i + H, i:i + W].permute(1, 2, 0) * 255).to(torch.uint8).contiguous().to(DEV) for i in range(CUT)]
    return out


@pytest.mark.parametrize("K", [1, 3])
def test_two_shots_through_r(K):
    m = make_model("R")
    u8 = two_shots()
    out, calls, padded, conv = run(m, u8, 60, 24, K, A=360, S=7, threshold=27)
    assert conv.cuts == [CUT]
    assert not any((a, b) == (CUT - 1, CUT) for qs in calls for a, b, _ in qs)
    kept = kept_samples(60, 24, 10, 360, 7, cuts=(CUT,))
    for samples in kept:   # each output within one shot
        assert len({s[1] >= CUT for s in samples}) == 1
    ref = reference(m, u8, padded, calls, kept)
    assert len(out) == len(kept)
    for k, (o, r) in enumerate(zip(out, ref)):
        assert _close(o, r), (k, (o.int() - r.int()).abs().max().item())
