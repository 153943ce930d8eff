"""The reference's video driver (src/video_Nx.py) on the sm_90a engine: interpolate a directory of frames N times and write the
two videos it writes, `output.mp4` (each frame side by side with the original it follows) and `flow.mp4` (the colour-wheel picture
of the motion GIMM predicted for every interpolated frame).

    python scripts/video_nx.py --source-path frames/ --output-path out/ --N 8 [--ds-factor 0.5] [-m config.yaml] [-l ckpt.pth]

Frames are read in sorted order with cv2 (BGR converted to RGB, as PIL's convert("RGB") gives the reference).  Padding, the
interpolation, the uint8 conversion and the flow pictures run on the GPU (gimmvfi_b200.video.VideoInterpolator with
with_flow=True); only uint8 frames cross to the host.  The frame sequence is the reference's: the first frame doubled, for every
pair the N-1 interpolated frames next to the pair's first frame, then the pair's second frame doubled, the very last one
dropped (images[:-1]), at 2N fps.  --frames writes numbered PNGs into output/ and flow/ instead of videos; this is also what
happens to a video whose frames the reference hands to ffmpeg (max(height, width // 2) > 2048) when ffmpeg is not installed.
--scene-threshold T (off unless given): a pair whose scene-cut score (gimmvfi_b200.video.scene_scores) is >= T is a hard cut and is
not interpolated; its N-1 frames are the nearer original and its flow pictures those of a zero flow, and the cuts are listed at the
end.  Without -l the model has seeded weights."""
import argparse
import os
import shutil
import subprocess
import sys
import tempfile

import cv2
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gimmvfi_b200 import create_model, load_config  # noqa: E402
from gimmvfi_b200.video import VideoInterpolator  # noqa: E402


def parse_args(argv=None):
    p = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    p.add_argument("-m", "--model-config", default=os.path.join(ROOT, "configs", "gimmvfi", "gimmvfi_r_arb.yaml"))
    p.add_argument("-l", "--load-path", default="", help="checkpoint with a 'state_dict' entry; seeded weights without it")
    p.add_argument("--source-path", required=True)
    p.add_argument("--output-path", required=True)
    p.add_argument("--N", type=int, default=8)
    p.add_argument("--ds-factor", type=float, default=1.0)
    p.add_argument("--frames", action="store_true", help="write PNG sequences output/%%04d.png and flow/%%04d.png instead of videos")
    p.add_argument("--pairs-per-call", type=int, default=1,
                   help="interpolate K consecutive pairs per engine call, each frame encoded once (1: one call per pair)")
    p.add_argument("--scene-threshold", type=float, default=None,
                   help="do not interpolate across a scene cut: a pair scoring >= this is one (27 is PySceneDetect's default); off if not given")
    return p.parse_args(argv)


class FrameSink:
    """video_Nx.py:53-84 images_to_video, fed frame by frame: cv2's mp4v writer, or ffmpeg on a PNG sequence for frames larger
    than 2048 pixels, or the PNG sequence itself (png_dir) when asked for or when ffmpeg is missing"""

    def __init__(self, video_path, png_dir, fps, force_png):
        self.video_path, self.png_dir, self.fps, self.force_png = video_path, png_dir, fps, force_png
        self.writer, self.tmp, self.dir, self.count = None, None, None, 0

    def write(self, img):
        if self.count == 0:
            h, w = img.shape[:2]
            big = max(h, w // 2) > 2048   # the reference's test, applied to every video it writes
            if self.force_png or (big and shutil.which("ffmpeg") is None):
                if big and not self.force_png:
                    print("%s: frames of %dx%d need ffmpeg, which is not installed: writing PNG frames to %s" % (
                        os.path.basename(self.video_path), w, h, self.png_dir))
                self.dir = self.png_dir
            elif big:
                self.tmp = self.dir = tempfile.mkdtemp(prefix="frames_", dir=os.path.dirname(self.video_path))
            else:
                self.writer = cv2.VideoWriter(self.video_path, cv2.VideoWriter_fourcc(*"mp4v"), self.fps, (w, h))
            if self.dir:
                os.makedirs(self.dir, exist_ok=True)
        if self.writer is not None:
            self.writer.write(img)
        else:
            cv2.imwrite(os.path.join(self.dir, "%04d.png" % self.count), img)
        self.count += 1

    def close(self):
        if self.writer is not None:
            self.writer.release()
        if self.tmp is not None:
            subprocess.run(["ffmpeg", "-framerate", str(self.fps), "-i", os.path.join(self.tmp, "%04d.png"), "-c:v", "libx264",
                            "-pix_fmt", "yuv420p", self.video_path], check=True)
            shutil.rmtree(self.tmp)


def build_model(args, dev):
    model, _ = create_model(load_config(args.model_config).arch)
    if args.load_path:
        ckpt = torch.load(args.load_path, map_location="cpu")
        model.load_state_dict(ckpt["state_dict"], strict=True)
    return model.to(dev).eval()


def main(argv=None):
    args = parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("video_nx.py needs a CUDA device")
    dev = torch.device("cuda")
    names = sorted(os.listdir(args.source_path))
    if len(names) < 2:
        raise SystemExit("video_nx.py: %s holds %d frame(s); at least 2 are needed" % (args.source_path, len(names)))
    os.makedirs(args.output_path, exist_ok=True)
    model = build_model(args, dev)
    fps = args.N * 2
    out = FrameSink(os.path.join(args.output_path, "output.mp4"), os.path.join(args.output_path, "output"), fps, args.frames)
    flow = FrameSink(os.path.join(args.output_path, "flow.mp4"), os.path.join(args.output_path, "flow"), fps, args.frames)
    ds = None if args.ds_factor == 1.0 else args.ds_factor   # a resize by 1 is the identity
    vi = VideoInterpolator(model, N=args.N, ds_factor=ds, bgr=True, with_flow=True, pairs_per_call=args.pairs_per_call,
                           scene_threshold=args.scene_threshold)
    host = lambda x: x.cpu().numpy()
    waiting = []   # originals whose interpolated frames have not come back yet (pairs_per_call > 1), oldest first
    per_pair = args.N - 1

    def emit(frames, flows, last):
        # frames / flows: N-1 per pair, in clip order; the pair from waiting[k] to waiting[k + 1]
        for k in range(len(frames) // per_pair if per_pair else 0):
            prev = waiting.pop(0)
            for fr, fl in zip(frames[k * per_pair:(k + 1) * per_pair], flows[k * per_pair:(k + 1) * per_pair]):
                out.write(host(torch.cat([prev, fr], 1)))
                flow.write(host(fl))
            if len(waiting) > 1 or not last:   # the reference appends every original twice-wide and drops the last image
                out.write(host(torch.cat([waiting[0], waiting[0]], 1)))

    for j, name in enumerate(names):
        bgr = cv2.imread(os.path.join(args.source_path, name), cv2.IMREAD_COLOR)
        if bgr is None:
            raise SystemExit("video_nx.py: cannot read %s" % name)
        cur_bgr = torch.from_numpy(bgr).to(dev)
        last = j == len(names) - 1
        if j == 0 and not last:   # (the reference drops the last image: a one-image input writes nothing)
            out.write(host(torch.cat([cur_bgr, cur_bgr], 1)))
        waiting.append(cur_bgr)
        frames, flows = vi.push(cur_bgr.flip(-1).contiguous())   # RGB in; frames come back BGR
        emit(frames, flows, last)
        if last:
            emit(*vi.flush(), last)
        print("frame %d / %d" % (j + 1, len(names)), flush=True)
    out.close()
    flow.close()
    print("wrote %d frames and %d flow pictures to %s" % (out.count, flow.count, args.output_path))
    if args.scene_threshold is not None:
        print("scene cuts (input frame j starts a new shot): %s" % (vi.cuts,))


if __name__ == "__main__":
    main()
