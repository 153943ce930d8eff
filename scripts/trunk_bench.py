"""The final decoder trunk's 3x3 256-channel half convolutions (ResBlock conv1 / conv3 / conv5, fi_components.py:97-154) through
gimmvfi_op_conv2d_wide and gimmvfi_op_conv2d_tc_f16 on the same inputs, alternated round by round, at the sizes the headline
configurations run them: pair1080 (1088x1920) and f2k (GIMM-VFI-F on a 2048x1080 pair at ds_factor 0.5: 544x1024).  With --base the
tc_f16 op of a second library (a parent build) joins the rotation.  Per layer class and arm: median and spread in ms over the rounds
(CUDA events around --reps calls), algorithmic TFLOP/s, the L2 -> SM bytes the kernel's tiles load (computed from the tile shapes below,
not measured) and those bytes over the time; per class max|wide - tc_f16| of the stored halves.  Prints the card and its power limit.

    python scripts/trunk_bench.py [--lib A.so] [--base B.so] [--rounds 7] [--reps 10]
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

ACT_PRELU = 3
SIZES = [("pair1080", 1088, 1920), ("f2k", 544, 1024)]
FORMS = ["conv1 256h>256h", "conv3 192h@256+64h>256h", "conv5 192h@256+64h>256h +res in place"]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def l2_bytes(kind, h, w, cin=256, cout=256):
    """bytes TMA moves from L2 into shared memory for one layer"""
    kb = cin // 64
    if kind == "wide":   # per (8x16 pixel tile, 128-channel N tile) and 64-channel K block: 3 halo copies {64, 8, 18} + 9 weight boxes {64, 128}
        tiles = ((w + 7) // 8) * ((h + 15) // 16) * (cout // 128)
        return tiles * kb * (3 * 8 * 18 * 128 + 9 * 128 * 128)
    # conv_tc f16, N = 128: per (16x8 pixel tile, N tile) and (tap, K block): an activation box {64, 16, 8} + a weight box {64, 128}
    tiles = ((w + 15) // 16) * ((h + 7) // 8) * (cout // 128)
    return tiles * 9 * kb * (16 * 8 * 128 + 128 * 128)


def view(t, c, off=0):
    n, h, w, ld = t.shape
    return View(t.data_ptr() + t.element_size() * off, n, h, w, c, ld, h * w * ld)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=DEFAULT_LIB)
    ap.add_argument("--base", default="", help="a parent library whose tc_f16 op joins the rotation")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("trunk_bench.py needs a CUDA device")
    lib = Lib(args.lib)
    arms = []
    if hasattr(lib.dll, "gimmvfi_op_conv2d_wide"):
        arms.append(("wide", "wide", lib))
    arms.append(("tc_f16", "tc", lib))
    if args.base:
        arms.append(("tc_f16 base", "tc", Lib(args.base)))
    name, limits = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, limits), flush=True)
    print("arms: %s" % ", ".join(a for a, _, _ in arms), flush=True)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    g = torch.Generator().manual_seed(0)
    P = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
    for size, H, W in SIZES:
        for form in FORMS:
            x = torch.randn(1, H, W, 256, generator=g).half().cuda()     # conv1's input; conv3 / conv5: channels 0-191 of it
            s = torch.randn(1, H, W, 64, generator=g).half().cuda()      # the 64-channel side output
            res0 = torch.randn(1, H, W, 256, generator=g).half().cuda()
            wt = torch.randn(256, 256, 3, 3, generator=g) / (256 * 9) ** 0.5
            w_h = wt.permute(2, 3, 0, 1).reshape(9, 256, 256).half().contiguous().cuda()   # [tap][cout][cin], as the engine packs w_tc_h
            w_dummy = torch.zeros(2 * 9 * 256 * 256, device="cuda")   # the op's fp32 weights: not read by the half path
            b = torch.zeros(288)
            b[:256] = 0.1 * torch.randn(256, generator=g)
            b = b.cuda()
            slope = (0.25 + 0.1 * torch.randn(256, generator=g)).cuda()
            two = not form.startswith("conv1")
            inplace = form.startswith("conv5")
            out = res0.clone() if inplace else torch.empty(1, H, W, 256, dtype=torch.float16, device="cuda")
            v0 = view(x, 192 if two else 256)
            v1 = view(s, 64) if two else None
            vo = view(out, 256)
            vr = vo if inplace else None
            act1, act2 = (0, ACT_PRELU) if inplace else (ACT_PRELU, 0)
            mask = 1 | 2 | (4 if inplace else 0)

            def call(kind, L):
                if kind == "wide":
                    L.check(L.dll.gimmvfi_op_conv2d_wide(C.byref(v0), C.byref(v1) if v1 else None, P(w_h), P(b), 256, 256, act1, P(slope),
                                                         C.byref(vr) if vr else None, act2, P(slope), mask, C.byref(vo), stream))
                else:
                    L.check(L.dll.gimmvfi_op_conv2d_tc_f16(C.byref(v0), C.byref(v1) if v1 else None, P(w_h), P(w_dummy), P(b), 256, 256, 3, 3,
                                                           act1, P(slope), C.byref(vr) if vr else None, act2, P(slope), mask, C.byref(vo),
                                                           stream))

            results = {}
            for arm, kind, L in arms:   # warm-up and each arm's result from the same inputs
                if inplace:
                    out.copy_(res0)
                call(kind, L)
                torch.cuda.synchronize()
                results[arm] = out.clone()
                call(kind, L)
            times = {arm: [] for arm, _, _ in arms}
            for _ in range(args.rounds):
                for arm, kind, L in arms:
                    if inplace:
                        out.copy_(res0)   # (values stay bounded over the repetitions; outside the timed window)
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.reps):
                        call(kind, L)
                    e1.record()
                    torch.cuda.synchronize()
                    times[arm].append(e0.elapsed_time(e1) / args.reps)
            flop = 2.0 * H * W * 256 * 256 * 9
            label = "%s %dx%d %s" % (size, H, W, form)
            meds = {}
            for arm, kind, _ in arms:
                t = times[arm]
                med = meds[arm] = statistics.median(t)
                nb = l2_bytes(kind, H, W)
                print("%-58s %-11s %7.3f ms [%.3f .. %.3f]  %6.1f TFLOP/s  L2->SM %5.1f GB  %5.2f TB/s"
                      % (label, arm, med, min(t), max(t), flop / med / 1e9, nb / 1e9, nb / med / 1e9), flush=True)
            if "wide" in results:
                d = (results["wide"].float() - results["tc_f16"].float()).abs().max().item()
                print("%-58s speed-up wide vs tc_f16 %.2fx  max|wide - tc_f16| = %.3e" % (label, meds["tc_f16"] / meds["wide"], d), flush=True)
            if args.base:
                eq = torch.equal(results["tc_f16"], results["tc_f16 base"])
                print("%-58s tc_f16 lib vs base bit-equal: %s" % (label, eq), flush=True)
            del x, s, res0, out, w_h, w_dummy


if __name__ == "__main__":
    main()
