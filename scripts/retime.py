"""Convert a directory of frames to another frame rate on the sm_90a engine: every output frame at input time k * fps_in / fps_out,
interpolated by GIMM-VFI where that time falls between two input frames, the input frame itself where it falls on one.

    python scripts/retime.py --source-path frames/ --output-path out/ --fps-in 24 --fps-out 60 [--ds-factor 0.5] [--pairs-per-call 4]
                             [--scene-threshold 27] [--shutter-angle 180 [--shutter-samples 7]] [--frames] [-m config.yaml]
                             [-l ckpt.pth]

Rates are exact rationals: 24, 30000/1001 or 29.97.  Frames are read in sorted order with cv2 (BGR converted to RGB); padding, the
interpolation and the uint8 conversion run on the GPU (gimmvfi_b200.video.FrameRateConverter), K pairs per engine call.  Writes
output.mp4 at fps_out, or numbered PNGs in output/ with --frames (and for frames larger than 2048 pixels when ffmpeg is missing, as
video_nx.py).  --scene-threshold T: a pair of consecutive input frames whose scene-cut score (gimmvfi_b200.video.scene_scores) is
>= T is a hard cut and is not interpolated; its output instants show the nearer input frame, and the cuts are listed at the end.
Off unless given.  --shutter-angle A: motion blur, each output frame the mean of --shutter-samples S (odd, default 7) sub-frames spread
over an exposure of A / 360 of an output frame interval centred on its instant (FrameRateConverter's shutter_angle); off unless given.
Without -l the model has seeded weights."""
import argparse
import os
import sys

import cv2
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gimmvfi_b200.video import FrameRateConverter  # noqa: E402
from video_nx import FrameSink, build_model  # noqa: E402


def parse_args(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    p.add_argument("-m", "--model-config", default=os.path.join(ROOT, "configs", "gimmvfi", "gimmvfi_r_arb.yaml"))
    p.add_argument("-l", "--load-path", default="", help="checkpoint with a 'state_dict' entry; seeded weights without it")
    p.add_argument("--source-path", required=True)
    p.add_argument("--output-path", required=True)
    p.add_argument("--fps-in", required=True, help="input frame rate: 24, 30000/1001, 29.97, ...")
    p.add_argument("--fps-out", required=True, help="output frame rate, as --fps-in")
    p.add_argument("--ds-factor", type=float, default=1.0)
    p.add_argument("--pairs-per-call", type=int, default=1,
                   help="frame pairs interpolated per engine call, each frame encoded once (the workspace grows with it)")
    p.add_argument("--frames", action="store_true", help="write a PNG sequence output/%%04d.png instead of output.mp4")
    p.add_argument("--scene-threshold", type=float, default=None,
                   help="do not interpolate across a scene cut: a pair scoring >= this is one (27 is PySceneDetect's default); off if not given")
    p.add_argument("--shutter-angle", type=float, default=None,
                   help="motion blur: the exposure of each output frame in degrees of its interval, in (0, 360] (180 is a film camera's); off "
                        "if not given")
    p.add_argument("--shutter-samples", type=int, default=7, help="sub-frames averaged per output frame with --shutter-angle (odd, 1 .. 63)")
    return p.parse_args(argv)


def main(argv=None):
    args = parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("retime.py needs a CUDA device")
    dev = torch.device("cuda")
    names = sorted(os.listdir(args.source_path))
    if not names:
        raise SystemExit("retime.py: %s holds no frames" % args.source_path)
    os.makedirs(args.output_path, exist_ok=True)
    model = build_model(args, dev)
    ds = None if args.ds_factor == 1.0 else args.ds_factor   # a resize by 1 is the identity
    conv = FrameRateConverter(model, args.fps_in, args.fps_out, ds_factor=ds, bgr=True, pairs_per_call=args.pairs_per_call,
                              scene_threshold=args.scene_threshold, shutter_angle=args.shutter_angle,
                              shutter_samples=args.shutter_samples)
    out = FrameSink(os.path.join(args.output_path, "output.mp4"), os.path.join(args.output_path, "output"), float(conv.fps_out), args.frames)
    for j, name in enumerate(names):
        bgr = cv2.imread(os.path.join(args.source_path, name), cv2.IMREAD_COLOR)
        if bgr is None:
            raise SystemExit("retime.py: cannot read %s" % name)
        for fr in conv.push(torch.from_numpy(bgr).to(dev).flip(-1).contiguous()):   # RGB in; frames come back BGR
            out.write(fr.cpu().numpy())
        print("frame %d / %d" % (j + 1, len(names)), flush=True)
    for fr in conv.flush():
        out.write(fr.cpu().numpy())
    out.close()
    print("wrote %d frames at %s fps to %s" % (out.count, conv.fps_out, args.output_path))
    if args.scene_threshold is not None:
        print("scene cuts (input frame j starts a new shot): %s" % (conv.cuts,))


if __name__ == "__main__":
    main()
