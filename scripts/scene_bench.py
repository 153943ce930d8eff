"""Scene-cut detection on the GPU: the speed of gimmvfi_op_scene_sums and scene_scores, and what detection costs a frame-rate conversion.

1. The op at 1920x1080 and 3840x2160 with n = 1 and n = 16 pairs, the pairs (a[i], b[i]) taken from two separate stacks.  Each timed
   window runs --iters launches between two CUDA events, cycling over as many independent buffer sets as it takes to exceed 256 MB, so
   no launch finds its frames in the 50 MB L2.  Reported: the median of --reps windows per launch, the bytes the op must read (6 per
   pixel per pair), the achieved GB/s, and the share of the 3.35 TB/s HBM3 bound (bytes / 3.35 TB/s over the time); then the same
   over the kernels' own device time from a torch.profiler pass of its own (kernel_*), which leaves out the host's launch gaps.
2. scene_scores on F = n + 1 frames: one launch on the views frames[:-1] and frames[1:] plus the read back, host clock around a
   synchronised call.
3. FrameRateConverter 24 -> 60 with GIMM-VFI-R on a seeded 1080p clip (--frames frames, --K pairs per call), without and with
   scene_threshold 27, alternating round by round after one warm-up pass each: device-timed ms per output frame and the difference.

Prints the card's name and power limit, read in the same run, and one JSON line per measurement.  Seeded weights and frames."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from gimmvfi_b200.video import FrameRateConverter, _scene_sums, scene_scores  # noqa: E402
from retime_bench import clip_u8, gpu_info, make_model  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet
SIZES = {"1080p": (1080, 1920), "2160p": (2160, 3840)}


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def bench_op(h, w, n, iters, reps, dev):
    bytes_per_call = n * h * w * 6
    sets = max(2, -(-(256 << 20) // bytes_per_call))
    g = torch.Generator(device=dev).manual_seed(h + n)
    bufs = [(torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device=dev, generator=g),
             torch.randint(0, 256, (n, h, w, 3), dtype=torch.uint8, device=dev, generator=g)) for _ in range(sets)]
    for a, b in bufs:   # warm-up
        _scene_sums(a, b)
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for i in range(iters):
            a, b = bufs[i % sets]
            _scene_sums(a, b)
        e.record()
        torch.cuda.synchronize()
        ms.append(s.elapsed_time(e) / iters)
    t = median(ms) * 1e-3
    # the kernels' own device time, from a profiled pass of its own: at small n the event window above also holds host launch gaps
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for i in range(iters):
            a, b = bufs[i % sets]
            _scene_sums(a, b)
        torch.cuda.synchronize()
    kern = [e for e in prof.key_averages() if "scene_sums" in e.key]
    k_us = sum(e.device_time_total for e in kern) / max(1, sum(e.count for e in kern))
    frames = torch.cat([bufs[0][0], bufs[0][1][-1:]], 0).contiguous()
    scene_scores(frames)
    host = []
    for _ in range(reps * 5):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        scene_scores(frames)
        host.append((time.perf_counter() - t0) * 1e3)
    return dict(size="%dx%d" % (w, h), n=n, buffer_sets=sets, us_per_launch=round(t * 1e6, 2), us_min=round(min(ms) * 1e3, 2),
                us_max=round(max(ms) * 1e3, 2), bytes=bytes_per_call, gb_per_s=round(bytes_per_call / t / 1e9, 1),
                share_of_hbm_bound=round(bytes_per_call / HBM_BYTES_PER_S / t, 3), hbm_bound_us=round(bytes_per_call / HBM_BYTES_PER_S * 1e6, 2),
                kernel_us=round(k_us, 2), kernel_gb_per_s=round(bytes_per_call / (k_us * 1e-6) / 1e9, 1) if k_us else None,
                kernel_share_of_hbm_bound=round(bytes_per_call / HBM_BYTES_PER_S / (k_us * 1e-6), 3) if k_us else None,
                scene_scores_ms=round(median(host), 3))


def bench_converter(frames_n, K, reps, dev):
    model = make_model("R", dev)
    frames = clip_u8(frames_n, 1080, 1920, dev, seed=1)

    def run(thr):
        conv = FrameRateConverter(model, 24, 60, pairs_per_call=K, scene_threshold=thr)
        out = []
        for f in frames:
            out += conv.push(f)
        out += conv.flush()
        return out, conv.cuts

    variants = {"off": None, "threshold27": 27}
    outs = {name: run(thr) for name, thr in variants.items()}   # warm-up
    torch.cuda.synchronize()
    ms = {name: [] for name in variants}
    for _ in range(reps):
        for name, thr in variants.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            out, _ = run(thr)
            e.record()
            torch.cuda.synchronize()
            ms[name].append(s.elapsed_time(e) / len(out))
    diff = max((x.int() - y.int()).abs().max().item() for x, y in zip(outs["off"][0], outs["threshold27"][0]))
    off, on = median(ms["off"]), median(ms["threshold27"])
    return dict(workload="FrameRateConverter 24->60 GIMM-VFI-R 1920x1080", frames=frames_n, outputs=len(outs["off"][0]), K=K,
                ms_per_frame_off=round(off, 3), ms_per_frame_threshold27=round(on, 3),
                range_off=[round(min(ms["off"]), 3), round(max(ms["off"]), 3)],
                range_threshold27=[round(min(ms["threshold27"]), 3), round(max(ms["threshold27"]), 3)],
                detection_cost_pct=round(100 * (on - off) / off, 2), cuts=outs["threshold27"][1], max_uint8_diff=diff)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frames", type=int, default=25)
    ap.add_argument("--K", type=int, default=1)
    ap.add_argument("--conv-reps", type=int, default=3)
    ap.add_argument("--skip-converter", action="store_true")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("scene_bench.py needs a CUDA device")
    dev = torch.device("cuda")
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for name, (h, w) in SIZES.items():
        for n in (1, 16):
            print(json.dumps(bench_op(h, w, n, args.iters if n == 1 else max(20, args.iters // 8), args.reps, dev)), flush=True)
    torch.cuda.empty_cache()
    if not args.skip_converter:
        print(json.dumps(bench_converter(args.frames, args.K, args.conv_reps, dev)), flush=True)


if __name__ == "__main__":
    main()
