"""Frames per second of a clip through VideoInterpolator: today's per-pair calls (pairs_per_call 1, GIMM-VFI-R's frame cache included)
against clip calls of K pairs (model.interpolate, each frame encoded once), for GIMM-VFI-R and -F at several frame sizes and N.

Every setting runs the same synthetic clip of --frames uint8 frames (on the device), once to warm up and then --reps timed passes, each
with a device synchronise before the clock stops; frames/s counts the interpolated frames, reported as the median and the range of the
passes.  The workspace bytes of one K-pair call (planned in the model's precision mode) are printed beside it; a
setting whose workspace does not fit the device is reported and skipped.  One JSON line per setting, plus the GPU's name and power
limit.  Seeded weights (the speed does not depend on them)."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from gimmvfi_b200 import GIMMVFI_R  # noqa: E402
from gimmvfi_b200.model_f import GIMMVFI_F  # noqa: E402
from gimmvfi_b200.video import InputPadder, VideoInterpolator  # noqa: E402
from gimmvfi_b200.weights import random_state_dict, random_state_dict_f  # noqa: E402

SIZES = {"256x448": (256, 448), "720p": (720, 1280), "1080p": (1080, 1920)}


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
    return m


def clip_u8(n, h, w, dev, seed=0):
    """n frames of a smooth pattern moving a few pixels per frame"""
    g = torch.Generator(device="cpu").manual_seed(seed)
    base = torch.rand(3, h // 16 + 4, w // 16 + 4, generator=g)
    big = torch.nn.functional.interpolate(base[None], size=(h + 64, w + 64), mode="bicubic", align_corners=False)[0].clamp(0, 1)
    return [(big[:, 3 * j:3 * j + h, 2 * j:2 * j + w].permute(1, 2, 0) * 255).to(torch.uint8).contiguous().to(dev) for j in range(n)]


def run_clip(model, frames, N, K):
    vi = VideoInterpolator(model, N=N, pairs_per_call=K)
    out = []
    for f in frames:
        out += vi.push(f)
    out += vi.flush()
    return len(out)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--models", default="R,F")
    ap.add_argument("--sizes", default=",".join(SIZES))
    ap.add_argument("--N", default="2,8")
    ap.add_argument("--K", default="1,2,4,8", help="pairs per call; 1 = per-pair calls")
    ap.add_argument("--frames", type=int, default=9)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default="", help="also append the JSON lines to this file")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("clip_bench.py needs a CUDA device")
    dev = torch.device("cuda")
    info = {"gpu": gpu_info()}
    print(json.dumps(info), flush=True)
    lines = [info]
    total = torch.cuda.get_device_properties(dev).total_memory
    for kind in args.models.split(","):
        model = make_model(kind, dev)
        model._ready(torch.empty(1, device=dev))   # the model's precision mode on its engine before the first plan
        for size in args.sizes.split(","):
            h, w = SIZES[size]
            frames = clip_u8(args.frames, h, w, dev)
            H, W = InputPadder((h, w), 32).padded_shape
            for N in (int(x) for x in args.N.split(",")):
                for K in (int(x) for x in args.K.split(",")):
                    rec = dict(model=kind, size=size, N=N, pairs_per_call=K, frames=args.frames)
                    if K == 1:
                        rec["workspace_bytes"] = model.engine.workspace_bytes(1, H, W, N - 1, None, H, W)
                    else:
                        rec["workspace_bytes"] = model.engine.clip_workspace_bytes(K + 1, [(i, i + 1) for i in range(K)], H, W, N - 1, None, H, W)
                    if rec["workspace_bytes"] > 0.85 * total:
                        rec["skipped"] = "workspace larger than the device"
                        print(json.dumps(rec), flush=True)
                        lines.append(rec)
                        continue
                    try:
                        run_clip(model, frames, N, K)   # warm-up
                        torch.cuda.synchronize()
                    except RuntimeError as ex:   # an allocation the plan did not foresee (torch's own buffers): reported
                        rec["error"] = str(ex).splitlines()[0][:200]
                    if "error" not in rec:
                        fps = []
                        for _ in range(args.reps):
                            t0 = time.perf_counter()
                            n = run_clip(model, frames, N, K)
                            torch.cuda.synchronize()
                            fps.append(n / (time.perf_counter() - t0))
                        fps.sort()
                        rec.update(interpolated_per_rep=n, fps_median=round(fps[len(fps) // 2], 2), fps_min=round(fps[0], 2),
                                   fps_max=round(fps[-1], 2))
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
