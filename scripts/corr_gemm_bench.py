"""All-pairs correlation in the 3xF16 form through gimmvfi_op_corr_volume_tc(split=1), two libraries alternated round by round: the
level-0 volumes of RAFT's pyramid at pair1080 (136x240 features) and batch720 (92x160), and FlowFormer's f2k cost volume (68x128),
C = 256.  One call is the operand split plus the GEMM.  Per shape: median and spread in ms over the rounds (CUDA events around
--reps calls), executed TFLOP/s (3 f16 MMAs per product), written GB/s, and the share of the floor max(executed FLOP / 989 TFLOP/s,
written bytes / 3.35 TB/s) (H100 SXM data sheet, dense f16, 700 W).  Prints the card and its power limit.

    python scripts/corr_gemm_bench.py [--lib A.so] [--base B.so] [--rounds 7] [--reps 10]
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

from gimmvfi_b200._lib import DEFAULT_LIB, Lib, view_of  # noqa: E402

SHAPES = [("pair1080_level0", 136, 240), ("batch720_level0", 92, 160), ("f2k_cost_volume", 68, 128)]
CH = 256
PEAK_F16, PEAK_HBM = 989e12, 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=DEFAULT_LIB)
    ap.add_argument("--base", default="", help="a second library, alternated with --lib")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("corr_gemm_bench.py needs a CUDA device")
    libs = [("lib", Lib(args.lib))] + ([("base", Lib(args.base))] if args.base else [])
    name, limits = card()
    print("card: %s | power.limit, clocks.max.sm: %s" % (name, limits), flush=True)
    g = torch.Generator().manual_seed(0)
    for label, h, w in SHAPES:
        n = h * w
        fa = torch.randn(1, h, w, CH, generator=g).cuda()
        fb = torch.randn(1, h, w, CH, generator=g).cuda()
        vol = torch.empty(n, n, device="cuda")
        scratch = torch.empty(2 * n * CH + n + 2048, device="cuda")
        stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        va, vb = view_of(fa), view_of(fb)

        def call(lib):
            lib.check(lib.dll.gimmvfi_op_corr_volume_tc(C.byref(va), C.byref(vb), C.c_void_p(scratch.data_ptr()), C.c_void_p(vol.data_ptr()), 1,
                                                        stream))

        outs = {}
        for key, lib in libs:   # warm-up (module load, attributes) and the result of each library
            call(lib); call(lib)
            torch.cuda.synchronize()
            outs[key] = vol.clone()
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
        flop = 3 * 2.0 * n * n * CH
        wbytes = 4.0 * n * n
        floor_ms = 1e3 * max(flop / PEAK_F16, wbytes / PEAK_HBM)
        for key, _ in libs:
            t = times[key]
            med = statistics.median(t)
            print("%-16s %-4s  %8.3f ms  [%.3f .. %.3f]  %6.1f TFLOP/s executed  %7.1f GB/s written  floor %.3f ms (%.2fx)"
                  % (label, key, med, min(t), max(t), flop / med / 1e9, wbytes / med / 1e6, floor_ms, med / floor_ms), flush=True)
        if args.base:
            d = (outs["lib"] - outs["base"]).abs().max().item()
            print("%-16s max|lib - base| = %.3e%s" % (label, d, " (bit-equal)" if torch.equal(outs["lib"], outs["base"]) else ""), flush=True)


if __name__ == "__main__":
    main()
