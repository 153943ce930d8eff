"""csrc/conv_halo.cu at the pair1080 layer shapes, storage types and slice strides (GIMM's cnn_encoder, res_conv, the final decoder's
upsample branch and resblock side convolutions), and at ragged sizes.  Strict reference as test_conv_tc_gpu.test_conv2d_halo: an fp64
convolution of the operands as the tensor core sees them (halves, or TF32-truncated activations / RN weights).  The output buffer is
filled with a sentinel first: channels outside the output slice must come back unchanged."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

import gpu_ops as K
from gimmvfi_b200._lib import default_lib, view_of

pytestmark = pytest.mark.gpu
DEV = "cuda"
SENTINEL = -3.25

HALF, F32 = torch.float16, torch.float32

# name: cin, cout, k, n, H, W, input (dtype, channels of the buffer, offset), pre-padded, residual (dtype, channels, offset) or None,
#       output (dtype, channels, offset), act1, act2
LAYERS = {
    "enc_32h_32h": (32, 32, 3, 2, 1088, 1920, (HALF, 32, 0), False, None, (HALF, 32, 0), 2, 0),
    "enc_32h_32h_res": (32, 32, 3, 2, 1088, 1920, (HALF, 32, 0), False, (HALF, 32, 0), (HALF, 32, 0), 0, 2),
    "enc1_16f32_32h": (16, 32, 3, 2, 1088, 1920, (F32, 16, 0), False, None, (HALF, 32, 0), 2, 0),
    "up6_32h_64h": (32, 64, 3, 2, 1088, 1920, (HALF, 32, 0), False, None, (HALF, 64, 0), 2, 0),
    "up7_1x1_64h_64h": (64, 64, 1, 2, 1088, 1920, (HALF, 64, 0), False, None, (HALF, 64, 0), 2, 0),
    "side_64h_slice_256": (64, 64, 3, 1, 1088, 1920, (HALF, 256, 192), False, None, (HALF, 64, 0), 3, 0),
    "enc7_32h_16f32_x64": (32, 16, 3, 1, 1088, 1920, (HALF, 32, 0), True, None, (F32, 64, 16), 0, 0),
    "res5_64h_32f32_res": (64, 32, 3, 1, 1088, 1920, (HALF, 64, 0), True, (F32, 64, 32), (F32, 32, 0), 0, 0),
    # ragged: H not a multiple of 16, W not a multiple of 8
    "ragged_32h_32h_res_n2": (32, 32, 3, 2, 37, 29, (HALF, 32, 0), False, (HALF, 32, 0), (HALF, 32, 0), 2, 3),
    "ragged_16f32_32h_n1": (16, 32, 3, 1, 45, 19, (F32, 16, 0), False, None, (HALF, 32, 0), 1, 0),
    "ragged_64h_slice_n1": (64, 64, 3, 1, 50, 21, (HALF, 256, 192), False, None, (HALF, 64, 0), 3, 0),
    "ragged_32h_16f32_x64_n2": (32, 16, 3, 2, 23, 35, (HALF, 32, 0), True, None, (F32, 64, 48), 2, 0),
    "ragged_1x1_64h_48h_n2": (64, 48, 1, 2, 19, 13, (HALF, 64, 0), False, (HALF, 48, 0), (HALF, 48, 0), 0, 1),
    "ragged_64h_32f32_res_n2": (64, 32, 3, 2, 33, 27, (HALF, 64, 0), True, (F32, 64, 32), (F32, 32, 0), 2, 0),
}


def rnd(*s, seed=0, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*s, generator=g) * scale).to(DEV)


def act(a, v, slope):
    return {0: lambda t: t, 1: F.relu, 2: lambda t: F.leaky_relu(t, 0.1), 3: lambda t: F.prelu(t, slope.double())}[a](v)


@pytest.mark.parametrize("name", list(LAYERS))
def test_conv_halo_layer(name):
    cin, cout, k, n, H, W, (idt, ic, ioff), prepad, res_spec, (odt, oc, ooff), act1, act2 = LAYERS[name]
    lib = default_lib()
    ih, iw = (H + 2, W + 2) if prepad else (H, W)
    xbuf = rnd(n, ih, iw, ic, seed=1).to(idt)
    w = rnd(cout, cin, k, k, seed=2, scale=1.0 / (cin * k * k) ** 0.5)
    b = rnd(cout, seed=3, scale=0.1)
    bb = torch.zeros((K.tc_cout_pad(cout) + 31) // 32 * 32 + 128, device=DEV)
    bb[:cout] = b
    slope = 0.25 + 0.1 * rnd(cout, seed=4)
    rbuf = rnd(n, H, W, res_spec[1], seed=5).to(res_spec[0]) if res_spec else None
    out = torch.full((n, H, W, oc), SENTINEL, dtype=odt, device=DEV)
    half_in = idt == HALF
    pw_h = K.pack_weight_tc_f16(w) if half_in else None
    pw = None if half_in else K.pack_weight_tc(w)
    mask = (1 if half_in else 0) | (2 if odt == HALF else 0) | (4 if res_spec and res_spec[0] == HALF else 0)
    vx = view_of(xbuf, cin, ioff)
    vr = view_of(rbuf, cout, res_spec[2]) if res_spec else None
    vo = view_of(out, cout, ooff)
    P = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    lib.check(lib.dll.gimmvfi_op_conv2d_halo(C.byref(vx), P(pw_h), P(pw), P(bb), cin, cout, act1, P(slope), C.byref(vr) if vr is not None else None,
                                             act2, P(slope), mask, 2 if k == 1 else int(prepad), C.byref(vo),
                                             C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()

    x = K.nchw(xbuf[..., ioff:ioff + cin].float())
    if half_in:
        ref = F.conv2d(x.double(), w.half().double(), b.double(), padding=0 if prepad else k // 2)
    else:
        ref = F.conv2d(K.tf32_trunc(x).double(), K.tf32_rn(w).double(), b.double(), padding=0 if prepad else k // 2)
    ref = act(act1, ref, slope)
    if res_spec:
        ref = ref + K.nchw(rbuf[..., res_spec[2]:res_spec[2] + cout].double())
    ref = act(act2, ref, slope).float()
    got = K.nchw(out[..., ooff:ooff + cout].float())
    err = (got - ref).abs().max().item()
    tol = (1e-3 if half_in else 5e-5 + 2.0 ** -11) * max(1.0, ref.abs().max().item())
    print("halo layer", name, "err %.3e (tol %.1e)" % (err, tol))
    assert err <= tol
    outside = torch.cat([out[..., :ooff], out[..., ooff + cout:]], dim=-1)
    assert bool((outside == SENTINEL).all()), "channels outside the output slice were written"
