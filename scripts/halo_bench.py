"""The K-poor convolutions of the pair1080 headline (GIMM-VFI-R, one 1088x1920 pair) through gimmvfi_op_conv2d_halo, one row per layer
class, at the benchmark's shapes, storage types and slice strides.  With --base a second library is alternated round by round and the
whole output buffer of each class (the channels outside a slice included) is compared bit for bit.  Per class: median and spread in ms
over the rounds (CUDA events around --reps calls), achieved GB/s of the compulsory bytes (input once at storage precision, the residual,
the output's channels; halo rows not counted) and the share of the floor = those bytes / 3.35 TB/s (H100 SXM data sheet, 700 W).
Prints the card and its power limit.

    python scripts/halo_bench.py [--lib A.so] [--base B.so] [--rounds 7] [--reps 10]
"""
import argparse
import ctypes as C
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from gimmvfi_b200._lib import DEFAULT_LIB, Lib, View  # noqa: E402

PEAK_HBM = 3.35e12
H, W = 1088, 1920
ACT_LRELU, ACT_PRELU = 2, 3

# label, launches per step, n, cin, cout, k, input (dtype, ld, channel offset), pre-padded, residual dtype or None,
# output (dtype, ld, channel offset), act1
CLASSES = [
    ("cnn_encoder.1 16f32>32h", 1, 2, 16, 32, 3, (torch.float32, 16, 0), False, None, (torch.float16, 32, 0), ACT_LRELU),
    ("enc.layers.0/upsample 32h>32h", 6, 2, 32, 32, 3, (torch.float16, 32, 0), False, None, (torch.float16, 32, 0), ACT_LRELU),
    ("enc.layers.2 32h>32h +res", 3, 2, 32, 32, 3, (torch.float16, 32, 0), False, torch.float16, (torch.float16, 32, 0), 0),
    ("upsample.6 32h>64h", 1, 2, 32, 64, 3, (torch.float16, 32, 0), False, None, (torch.float16, 64, 0), ACT_LRELU),
    ("upsample.7 1x1 64h>64h", 1, 2, 64, 64, 1, (torch.float16, 64, 0), False, None, (torch.float16, 64, 0), ACT_LRELU),
    ("cnn_encoder.7 32h>16f32 X64", 2, 1, 32, 16, 3, (torch.float16, 32, 0), True, None, (torch.float32, 64, 16), 0),
    ("res_conv.1 32h>64h", 1, 1, 32, 64, 3, (torch.float16, 32, 0), False, None, (torch.float16, 64, 0), ACT_LRELU),
    ("res_conv.3.0 64h>64h", 1, 1, 64, 64, 3, (torch.float16, 64, 0), False, None, (torch.float16, 64, 0), ACT_LRELU),
    ("res_conv.3.2 64h>64h +res", 1, 1, 64, 64, 3, (torch.float16, 64, 0), False, torch.float16, (torch.float16, 64, 0), 0),
    ("res_conv.5 64h>32f32 +res", 1, 1, 64, 32, 3, (torch.float16, 64, 0), True, torch.float32, (torch.float32, 32, 0), 0),
    ("resblock conv2/4 64h[192:256]>64h", 6, 1, 64, 64, 3, (torch.float16, 256, 192), False, None, (torch.float16, 64, 0), ACT_PRELU),
]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def view(t, c, off):
    n, h, w, ld = t.shape
    return View(t.data_ptr() + t.element_size() * off, n, h, w, c, ld, h * w * ld)


def pack_f16(w):   # [taps][cout_pad][64] halves, as the engine packs them for conv_tc / conv_halo (cout_pad: cout to 16, cout <= 64)
    cout, cin, kh, kw = w.shape
    p = torch.zeros(kh * kw, (cout + 15) // 16 * 16, 64, dtype=torch.float16)
    p[:, :cout, :cin] = w.permute(2, 3, 0, 1).reshape(kh * kw, cout, cin).half()
    return p.cuda()


def pack_tf32(w):   # [taps][cout_pad][32] fp32, RN to TF32
    cout, cin, kh, kw = w.shape
    i = w.contiguous().view(torch.int32)
    hi = ((i + 0xFFF + ((i >> 13) & 1)) & ~0x1FFF).view(torch.float32)
    p = torch.zeros(kh * kw, (cout + 15) // 16 * 16, 32)
    p[:, :cout, :cin] = hi.permute(2, 3, 0, 1).reshape(kh * kw, cout, cin)
    return p.cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=DEFAULT_LIB)
    ap.add_argument("--base", default="", help="a second library, alternated with --lib")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("halo_bench.py needs a CUDA device")
    libs = [("lib", Lib(args.lib))] + ([("base", Lib(args.base))] if args.base else [])
    name, limits = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, limits), flush=True)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    g = torch.Generator().manual_seed(0)
    total = {key: 0.0 for key, _ in libs}
    total_floor = 0.0
    all_equal = True
    for label, per_step, n, cin, cout, k, (idt, ild, ioff), prepad, rdt, (odt, old, ooff), act1 in CLASSES:
        ih, iw = (H + 2, W + 2) if prepad else (H, W)
        x = torch.randn(n, ih, iw, ild, generator=g).to(idt).cuda()
        w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
        b = torch.zeros(128)
        b[:cout] = 0.1 * torch.randn(cout, generator=g)
        b = b.cuda()
        slope = (0.25 + 0.1 * torch.randn(128, generator=g)).cuda()
        res = torch.randn(n, H, W, cout, generator=g).to(rdt).cuda() if rdt is not None else None
        out = torch.full((n, H, W, old), 7.0, dtype=odt, device="cuda")   # sentinel in the channels outside the slice
        pw_h = pack_f16(w) if idt == torch.float16 else None
        pw = pack_tf32(w) if idt == torch.float32 else None
        vx, vo = view(x, cin, ioff), view(out, cout, ooff)
        vr = view(res, cout, 0) if res is not None else None
        mask = (1 if idt == torch.float16 else 0) | (2 if odt == torch.float16 else 0) | (4 if rdt == torch.float16 else 0)
        mode = 2 if k == 1 else int(prepad)

        def call(lib):
            lib.check(lib.dll.gimmvfi_op_conv2d_halo(
                C.byref(vx), C.c_void_p(pw_h.data_ptr()) if pw_h is not None else None, C.c_void_p(pw.data_ptr()) if pw is not None else None,
                C.c_void_p(b.data_ptr()),
                cin, cout, act1, C.c_void_p(slope.data_ptr()), C.byref(vr) if vr is not None else None, ACT_LRELU if res is not None else 0,
                C.c_void_p(slope.data_ptr()), mask, mode, C.byref(vo), stream))

        outs = {}
        for key, lib in libs:   # warm-up (module load, attributes) and the result of each library
            out.fill_(7.0)
            call(lib); call(lib)
            torch.cuda.synchronize()
            outs[key] = out.clone()
        times = {key: [] for key, _ in libs}
        for _ in range(args.rounds):
            for key, lib in libs:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.reps):
                    call(lib)
                e1.record()
                torch.cuda.synchronize()
                times[key].append(e0.elapsed_time(e1) / args.reps)
        px = n * H * W
        nbytes = px * (cin * x.element_size() + cout * out.element_size() + (cout * res.element_size() if res is not None else 0))
        floor_ms = 1e3 * nbytes / PEAK_HBM
        total_floor += per_step * floor_ms
        for key, _ in libs:
            t = times[key]
            med = statistics.median(t)
            total[key] += per_step * med
            print("%-34s x%d %-4s  %7.3f ms  [%.3f .. %.3f]  %6.0f GB/s  floor %.3f ms (%.2fx)"
                  % (label, per_step, key, med, min(t), max(t), nbytes / med / 1e6, floor_ms, med / floor_ms), flush=True)
        if args.base:
            eq = torch.equal(outs["lib"], outs["base"])
            all_equal &= eq
            d = (outs["lib"].float() - outs["base"].float()).abs().max().item()
            print("%-34s max|lib - base| = %.3e%s" % (label, d, " (bit-equal)" if eq else " (DIFFERENT)"), flush=True)
        del x, res, out
    for key, _ in libs:
        print("per step (launch counts as listed, full resolution): %-4s %.3f ms  floor %.3f ms (%.2fx)"
              % (key, total[key], total_floor, total[key] / total_floor))
    if args.base:
        print("all classes bit-equal: %s" % all_equal)


if __name__ == "__main__":
    main()
