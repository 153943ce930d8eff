"""Frame-rate conversion on the engine: FrameRateConverter with K pairs per interpolate_at call against the loop available without it,
one GIMMVFI forward per pair at that pair's own timesteps.

Workloads: a seeded synthetic clip of --frames frames at 1080p through GIMM-VFI-R, and at 2K (1080x2048) with ds_factor 0.5 through
GIMM-VFI-F, converted 24 -> 60 and 60 -> 24.  In one process, the variants (K in --K, and the per-pair loop) alternate round by round:
one warm-up pass each, then --reps timed passes, each between two CUDA events on the current stream with a synchronise after the
last.  Reported per variant: device-timed ms per output frame (median and range), the speed-up of the median against the loop, the
max |d imgt_pred| against the loop (float outputs of the same queries, before the uint8 conversion; the splat's float atomics make a
few 1e-6 normal), and the workspace bytes of one K-pair call; a K whose call does not fit the device is reported and skipped.  Prints the card's name and power limit, read in the same run, and
one JSON line per workload.  Seeded weights (the speed does not depend on them)."""
import argparse
import json
import math
import os
import subprocess
import sys
from fractions import Fraction

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from gimmvfi_b200 import GIMMVFI_R  # noqa: E402
from gimmvfi_b200.model_f import GIMMVFI_F  # noqa: E402
from gimmvfi_b200.video import FrameRateConverter, InputPadder  # noqa: E402
from gimmvfi_b200.weights import random_state_dict, random_state_dict_f  # noqa: E402

WORKLOADS = {"r1080": ("R", (1080, 1920), None), "f2k": ("F", (1080, 2048), 0.5)}


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except Exception as ex:   # (reported, not fatal)
        return "unknown (%s)" % ex


def make_model(kind, dev):
    if kind == "R":
        m = GIMMVFI_R(seed=0).to(dev).eval()
        m.load_state_dict(random_state_dict(0), strict=True)
    else:
        m = GIMMVFI_F(seed=0).to(dev).eval()
        m.load_state_dict(random_state_dict_f(0), strict=True)
    m.aux_outputs = False
    return m


def clip_u8(n, h, w, dev, seed=0):
    """n frames of a smooth pattern moving a few pixels per frame"""
    g = torch.Generator(device="cpu").manual_seed(seed)
    base = torch.rand(3, h // 16 + 4, w // 16 + 4, generator=g)
    big = torch.nn.functional.interpolate(base[None], size=(h + 4 * n, w + 4 * n), mode="bicubic", align_corners=False)[0].clamp(0, 1)
    return [(big[:, 3 * j:3 * j + h, 2 * j:2 * j + w].permute(1, 2, 0) * 255).to(torch.uint8).contiguous().to(dev) for j in range(n)]


def schedule(n, fps_in, fps_out):
    """FrameRateConverter's output instants over n frames: ("frame", j) or ("query", j - 1, j, t)"""
    step, out, k = Fraction(fps_in) / Fraction(fps_out), [], 0
    while k * step <= n - 1:
        tau = k * step
        a = math.floor(tau)
        out.append(("frame", a) if tau.denominator == 1 else ("query", a, a + 1, float(np.float32(float(tau - a)))))
        k += 1
    return out


def run_converter(model, frames, fps_in, fps_out, ds, K):
    conv = FrameRateConverter(model, fps_in, fps_out, ds_factor=ds, pairs_per_call=K)
    out = []
    for f in frames:
        out += conv.push(f)
    return out + conv.flush()


def pair_preds(model, padded, a, b, ts, ds):
    """imgt_pred (T,3,H,W) of forward() with B = 1 on one pair at its own timesteps"""
    H, W = padded.shape[-2:]
    xs = torch.stack([padded[a], padded[b]], 1).unsqueeze(0).contiguous()
    ratio = 1.0 if ds is None else ds
    coord = [(model.sample_coord_input(1, (H, W), [t], device=xs.device, upsample_ratio=ratio), None) for t in ts]
    tt = [t * torch.ones(1, device=xs.device) for t in ts]
    return torch.cat(model(xs, coord, t=tt, ds_factor=ds)["imgt_pred"], 0)


def run_loop(model, frames, sched, ds):
    """the per-pair loop: each pair with queries through one forward at its own timesteps; integral instants are the input frames"""
    padder = InputPadder(frames[0].shape[:2], 32)
    padded, out, j = {}, [], 0
    while j < len(sched):
        e = sched[j]
        if e[0] == "frame":
            out.append(frames[e[1]].flip(-1))
            j += 1
            continue
        a, b = e[1], e[2]
        mine = [x for x in sched[j:] if x[0] == "query" and x[1] == a]
        for f in (a, b):
            if f not in padded:
                padded[f] = padder.pad_u8(frames[f].unsqueeze(0))[0]
        x = torch.stack([padded[a], padded[b]], 0)
        out += list(padder.unpad_u8(pair_preds(model, x, 0, 1, [q[3] for q in mine], ds)).unbind(0))
        padded.pop(a, None)
        j += len(mine)
    return out


def max_delta(model, frames, sched, ds, K):
    """max |d imgt_pred| between interpolate_at calls of K pairs (as the converter makes them) and the per-pair forwards"""
    padder = InputPadder(frames[0].shape[:2], 32)
    qs = [e[1:] for e in sched if e[0] == "query"]
    pairs = sorted({(a, b) for a, b, _ in qs})
    worst = 0.0
    for c in range(0, len(pairs), K):
        chunk = pairs[c:c + K]
        used = sorted({f for p in chunk for f in p})
        local = {f: i for i, f in enumerate(used)}
        x = padder.pad_u8(torch.stack([frames[f] for f in used], 0))
        mine = [q for q in qs if (q[0], q[1]) in chunk]
        got = model._interpolate_at(x, [(local[a], local[b], t) for a, b, t in mine], ds, False)["imgt_pred"]
        for a, b in chunk:
            idx = [i for i, q in enumerate(mine) if (q[0], q[1]) == (a, b)]
            ref = pair_preds(model, x, local[a], local[b], [mine[i][2] for i in idx], ds)
            worst = max(worst, (got[idx] - ref).abs().max().item())
    return worst


def timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    n = len(fn())
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e), n


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--rates", default="24:60,60:24")
    ap.add_argument("--K", default="1,4,8")
    ap.add_argument("--frames", type=int, default=25)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("retime_bench.py needs a CUDA device")
    dev = torch.device("cuda")
    info = {"gpu": gpu_info()}
    print(json.dumps(info), flush=True)
    lines = [info]
    Ks = [int(k) for k in args.K.split(",")]
    total = torch.cuda.get_device_properties(dev).total_memory
    for wl in args.workloads.split(","):
        kind, (h, w), ds = WORKLOADS[wl]
        model = make_model(kind, dev)
        model._ready(torch.empty(1, device=dev))   # the model's precision mode on its engine before the first plan
        frames = clip_u8(args.frames, h, w, dev, seed=1)
        H, W = InputPadder((h, w), 32).padded_shape
        Hc, Wc = (H, W) if ds is None else (int(H * ds), int(W * ds))
        for rate in args.rates.split(","):
            fi, fo = (int(x) for x in rate.split(":"))
            sched = schedule(args.frames, fi, fo)
            qs = [e[1:] for e in sched if e[0] == "query"]
            pairs = sorted({(a, b) for a, b, _ in qs})
            rec = dict(workload=wl, model=kind, size="%dx%d" % (h, w), ds=ds, fps_in=fi, fps_out=fo, frames=args.frames,
                       outputs=len(sched), queries=len(qs), pairs_with_queries=len(pairs))
            variants = {}
            for K in Ks:
                chunk = pairs[:K]
                used = sorted({f for p in chunk for f in p})
                local = {f: i for i, f in enumerate(used)}
                mine = [(local[a], local[b], t) for a, b, t in qs if (a, b) in chunk]
                ws = model.engine.queries_workspace_bytes(len(used), mine, H, W, ds, Hc, Wc) if mine else 0
                if ws > 0.85 * total:   # (the volumes of K pairs: the call does not fit the device)
                    rec["K%d" % K] = dict(workspace_bytes=ws, skipped="workspace larger than the device")
                    continue
                variants["K%d" % K] = lambda K=K: run_converter(model, frames, fi, fo, ds, K)
                rec["K%d" % K] = dict(workspace_bytes=ws)
            variants["per_pair"] = lambda: run_loop(model, frames, sched, ds)
            for name, fn in variants.items():   # warm-up, every shape each variant uses
                fn()
            torch.cuda.synchronize()
            ms = {name: [] for name in variants}
            for _ in range(args.reps):
                for name, fn in variants.items():
                    t, n = timed(fn)
                    assert n == len(sched), (name, n, len(sched))
                    ms[name].append(t / n)
            base = sorted(ms["per_pair"])[len(ms["per_pair"]) // 2]
            for name, v in ms.items():
                v = sorted(v)
                med = v[len(v) // 2]
                r = rec.get(name, {})
                r.update(ms_per_frame=round(med, 3), ms_min=round(v[0], 3), ms_max=round(v[-1], 3), speedup=round(base / med, 3))
                if name != "per_pair":
                    r["max_abs_diff_imgt_pred"] = max_delta(model, frames, sched, ds, int(name[1:])) if qs else 0.0
                else:
                    T = max(sum(1 for q in qs if (q[0], q[1]) == p) for p in pairs) if qs else 1
                    r["workspace_bytes"] = model.engine.workspace_bytes(1, H, W, T, ds, Hc, Wc)
                rec[name] = r
            print(json.dumps(rec), flush=True)
            lines.append(rec)
            model.engine._ws = None
            torch.cuda.empty_cache()
        del model
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "a") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
