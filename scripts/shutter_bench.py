"""Shutter-angle motion blur in frame-rate conversion: FrameRateConverter with shutter_angle A and shutter_samples S against the same
converter without a shutter, and the blend op's own time.

Workloads: a seeded synthetic clip of --frames frames at 1080p through GIMM-VFI-R, and at 2K (1080x2048) with ds_factor 0.5 through
GIMM-VFI-F, converted 60 -> 24 with one pair per engine call.  In one process the variants (no shutter, and every A in --angles with
every S in --samples) alternate round by round: one warm-up pass each, then --reps timed passes, each between two CUDA events on the
current stream with a synchronise after the last.  Reported per variant: device-timed ms per output frame (median and range), queries
per output frame, and the workspace bytes of the largest engine call.  Then, in a separate torch.profiler pass per shutter variant,
the blend kernel (gimmvfi_op_blend_u8): its mean time per output frame, the bytes it must move (12 per pixel per engine sub-frame, 3 per
pixel per input frame and for the output, from the kept samples), its share of the HBM bound at 3.35 TB/s, and its share of the
variant's ms per output frame.  Prints the card's name and power limit, read in the same run, and one JSON line per workload.  Seeded
weights (the speed does not depend on them)."""
import argparse
import json
import math
import os
import sys
from fractions import Fraction

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from gimmvfi_b200.video import SNAP, FrameRateConverter, InputPadder  # noqa: E402
from retime_bench import clip_u8, gpu_info, make_model, timed  # noqa: E402

WORKLOADS = {"r1080": ("R", (1080, 1920), None), "f2k": ("F", (1080, 2048), 0.5)}
HBM = 3.35e12   # bytes/s, the H100 SXM data sheet's HBM3 bandwidth


def samples(n, fps_in, fps_out, A, S):
    """each output's samples inside the clip, ("frame", f) or ("query", a, a + 1, t) (no cuts, so every one is kept)"""
    step = Fraction(fps_in) / Fraction(fps_out)
    wnd = Fraction(A) / 360 * step
    outs, k = [], 0
    while k * step <= n - 1:
        cur = []
        for i in range(S):
            x = k * step - wnd / 2 + Fraction(2 * i + 1, 2 * S) * wnd
            if 0 <= x <= n - 1:
                a, off = math.floor(x), x - math.floor(x)
                cur.append(("frame", a) if off <= SNAP else ("frame", a + 1) if off >= 1 - SNAP else
                           ("query", a, a + 1, float(np.float32(float(off)))))
        outs.append(cur)
        k += 1
    return outs


def run(model, frames, ds, A, S):
    conv = FrameRateConverter(model, 60, 24, ds_factor=ds, pairs_per_call=1, shutter_angle=A, shutter_samples=S)
    out = []
    for f in frames:
        out += conv.push(f)
    return out + conv.flush()


def blend_us(model, frames, ds, A, S):
    """(mean device time of the blend kernel per launch in us, launches recorded), from a torch.profiler pass of its own"""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run(model, frames, ds, A, S)
        torch.cuda.synchronize()
    kern = [e for e in prof.key_averages() if "blend_u8_kernel" in e.key]
    launches = sum(e.count for e in kern)
    assert launches > 0, "no blend_u8_kernel in the trace"
    return sum(e.device_time_total for e in kern) / launches, launches


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--angles", default="180,360")
    ap.add_argument("--samples", default="3,7")
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("shutter_bench.py needs a CUDA device")
    dev = torch.device("cuda")
    info = {"gpu": gpu_info()}
    print(json.dumps(info), flush=True)
    lines = [info]
    shutters = [(int(a), int(s)) for a in args.angles.split(",") for s in args.samples.split(",")]
    for wl in args.workloads.split(","):
        kind, (h, w), ds = WORKLOADS[wl]
        model = make_model(kind, dev)
        model._ready(torch.empty(1, device=dev))   # the model's precision mode on its engine before the first plan
        frames = clip_u8(args.frames, h, w, dev, seed=1)
        H, W = InputPadder((h, w), 32).padded_shape
        Hc, Wc = (H, W) if ds is None else (int(H * ds), int(W * ds))
        rec = dict(workload=wl, model=kind, size="%dx%d" % (h, w), ds=ds, fps_in=60, fps_out=24, frames=args.frames)
        variants, sched = {"none": lambda: run(model, frames, ds, None, 7)}, {"none": samples(args.frames, 60, 24, 360, 1)}
        for A, S in shutters:
            variants["A%d_S%d" % (A, S)] = lambda A=A, S=S: run(model, frames, ds, A, S)
            sched["A%d_S%d" % (A, S)] = samples(args.frames, 60, 24, A, S)
        for name, fn in variants.items():   # warm-up, every shape each variant uses
            fn()
        torch.cuda.synchronize()
        ms = {name: [] for name in variants}
        for _ in range(args.reps):
            for name, fn in variants.items():
                t, n = timed(fn)
                assert n == len(sched[name]), (name, n, len(sched[name]))
                ms[name].append(t / n)
        for name, v in ms.items():
            v = sorted(v)
            outs = sched[name]
            qs = [s for o in outs for s in o if s[0] == "query"]
            per_pair = {}
            for q in qs:
                per_pair.setdefault(q[1:3], []).append((0, 1, q[3]))
            biggest = max(per_pair.values(), key=len) if per_pair else []
            r = dict(ms_per_frame=round(v[len(v) // 2], 3), ms_min=round(v[0], 3), ms_max=round(v[-1], 3),
                     queries_per_output=round(len(qs) / len(outs), 3),
                     workspace_bytes=model.engine.queries_workspace_bytes(2, biggest, H, W, ds, Hc, Wc) if biggest else 0)
            if name != "none":
                A, S = (int(x[1:]) for x in name.split("_"))
                us, launches = blend_us(model, frames, ds, A, S)
                nbytes = sum(h * w * (3 + sum(12 if s[0] == "query" else 3 for s in o)) for o in outs) / len(outs)
                r.update(blend_us=round(us, 2), blend_launches_traced=launches, blend_mb=round(nbytes / 1e6, 2),
                         blend_hbm_share=round(nbytes / HBM * 1e6 / us, 3), blend_share_of_frame=round(us / 1e3 / r["ms_per_frame"], 5))
            rec[name] = r
        print(json.dumps(rec), flush=True)
        lines.append(rec)
        del model
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "a") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
