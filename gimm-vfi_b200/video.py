"""GPU-side pre/post-processing of the reference's video driver (src/video_Nx.py:134-216) — SURVEY.md §8(f)
row 2.  uint8 frames go to the device once; /255, replicate-padding to a multiple of 32 (InputPadder,
src/utils/utils.py:156-185), the N-1 interpolations, un-padding and the uint8 (BGR) conversion all happen on
the GPU; only uint8 frames cross the PCIe bus."""
import ctypes as C
import math
import numbers
from fractions import Fraction
from typing import List, Optional

import numpy as np
import torch

from ._lib import GimmvfiError, default_lib


class InputPadder:
    """src/utils/utils.py:156-185 — same pad arithmetic, GPU kernels instead of F.pad / slicing."""

    def __init__(self, dims, divisor: int = 32):
        self.ht, self.wd = dims[-2:]
        pad_ht = (((self.ht // divisor) + 1) * divisor - self.ht) % divisor
        pad_wd = (((self.wd // divisor) + 1) * divisor - self.wd) % divisor
        self._pad = [pad_wd // 2, pad_wd - pad_wd // 2, pad_ht // 2, pad_ht - pad_ht // 2]

    @property
    def padded_shape(self):
        return self.ht + self._pad[2] + self._pad[3], self.wd + self._pad[0] + self._pad[1]

    def unpad_box(self, ht: int, wd: int):
        """InputPadder._unpad's crop of a (..., ht, wd) tensor as slice bounds (top, bottom, left, right).  The pad amounts are
        the frames' even when the tensor has another size: video_Nx.py:183 crops the network-resolution flowt this way, so at
        ds_factor < 1 the crop removes the full-resolution padding from a smaller picture."""
        return self._pad[2], ht - self._pad[3], self._pad[0], wd - self._pad[1]

    def pad_u8(self, frames_u8: torch.Tensor) -> torch.Tensor:
        """(n,h,w,3) uint8 RGB on the GPU -> (n,3,H,W) float32 in [0,1], replicate-padded."""
        assert frames_u8.is_cuda and frames_u8.dtype == torch.uint8 and frames_u8.dim() == 4 and frames_u8.shape[-1] == 3
        f = frames_u8.contiguous()
        n, h, w, _ = f.shape
        H, W = self.padded_shape
        out = torch.empty(n, 3, H, W, dtype=torch.float32, device=f.device)
        lib = default_lib()
        s = C.c_void_p(torch.cuda.current_stream(f.device).cuda_stream)
        lib.check(lib.dll.gimmvfi_op_frames_u8_to_padded_f32(C.c_void_p(f.data_ptr()), n, h, w, C.c_void_p(out.data_ptr()), H, W,
                                                             self._pad[2], self._pad[0], s))
        return out

    def unpad_u8(self, pred: torch.Tensor, bgr: bool = True) -> torch.Tensor:
        """(n,3,H,W) float32 -> (n,h,w,3) uint8, `(x*255).astype(uint8)`, BGR by default like video_Nx.py:190-196."""
        assert pred.is_cuda and pred.dtype == torch.float32 and pred.dim() == 4 and pred.shape[1] == 3
        p = pred.contiguous()
        n, _, H, W = p.shape
        out = torch.empty(n, self.ht, self.wd, 3, dtype=torch.uint8, device=p.device)
        lib = default_lib()
        s = C.c_void_p(torch.cuda.current_stream(p.device).cuda_stream)
        lib.check(lib.dll.gimmvfi_op_pred_to_u8(C.c_void_p(p.data_ptr()), n, H, W, C.c_void_p(out.data_ptr()), self.ht, self.wd,
                                                self._pad[2], self._pad[0], int(bgr), s))
        return out


def _scene_sums(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """gimmvfi_op_scene_sums on two contiguous (n,h,w,3) uint8 stacks on the device -> (n,3) int64 device tensor: the sums of |dH|,
    |dS|, |dV| of each pair (a[i], b[i]).  The op writes every sum."""
    n, h, w, _ = a.shape
    sums = torch.empty(n, 3, dtype=torch.int64, device=a.device)
    lib = default_lib()
    s = C.c_void_p(torch.cuda.current_stream(a.device).cuda_stream)
    lib.check(lib.dll.gimmvfi_op_scene_sums(C.c_void_p(a.data_ptr()), C.c_void_p(b.data_ptr()), n, h, w, C.c_void_p(sums.data_ptr()), s))
    return sums


def scores_from_sums(sums: torch.Tensor, h: int, w: int) -> torch.Tensor:
    """(n,3) integer sums on the host -> the n scores, float64: the exact integer total over one float64 division by 3 h w"""
    return sums.to(torch.int64).sum(1).to(torch.float64) / float(3 * h * w)


def scene_scores(frames_u8: torch.Tensor) -> torch.Tensor:
    """The scene-cut scores of consecutive frames: (F,h,w,3) uint8 RGB frames on the device, F >= 2, contiguous -> the F - 1 scores
    (float64, on the host), score j - 1 being that of (frames[j - 1], frames[j]).  The score is PySceneDetect's ContentDetector content
    value with HSV weights 1, 1, 1: both frames go to 8-bit HSV as cv2.cvtColor(x, cv2.COLOR_RGB2HSV) does, and the score is
    (sum |dH| + sum |dS| + sum |dV|) / (3 h w) over every pixel, H not wrapped.  A hard cut typically scores above 27 (PySceneDetect's
    default threshold for it), frames within a shot below.  One kernel over the views frames[:-1] and frames[1:], one read back."""
    if not torch.is_tensor(frames_u8) or not frames_u8.is_cuda:
        raise ValueError("scene_scores: frames must be a CUDA tensor")
    if frames_u8.dtype != torch.uint8 or frames_u8.dim() != 4 or frames_u8.shape[-1] != 3:
        raise ValueError("scene_scores: frames must be (F,h,w,3) uint8, got %s %s" % (tuple(frames_u8.shape), frames_u8.dtype))
    F, h, w, _ = frames_u8.shape
    if F < 2 or h < 1 or w < 1:
        raise ValueError("scene_scores: needs at least 2 frames of at least 1x1 pixels, got %s" % (tuple(frames_u8.shape),))
    if not frames_u8.is_contiguous():
        raise ValueError("scene_scores: the frame stack must be contiguous")
    return scores_from_sums(_scene_sums(frames_u8[:-1], frames_u8[1:]).cpu(), h, w)


def _pair_sums(a_u8: torch.Tensor, b_u8: torch.Tensor) -> torch.Tensor:
    """the (1,3) device sums of one pair of (h,w,3) uint8 frames, enqueued and not read"""
    return _scene_sums(a_u8.contiguous().unsqueeze(0), b_u8.contiguous().unsqueeze(0))


def _scene_threshold(x) -> Optional[float]:
    if x is None:
        return None
    if isinstance(x, bool) or not isinstance(x, numbers.Real) or not math.isfinite(x) or x <= 0:
        raise ValueError("scene_threshold must be None or a finite number > 0, got %r" % (x,))
    return float(x)


class _Cuts:
    """The scene-cut scores of a clip's consecutive input frames: the score of pair (j - 1, j) is enqueued on the device when frame j is
    pushed, and every waiting score is read back in one copy when a decision is due.  `cuts`: the j whose score was >= the threshold."""

    def __init__(self, threshold: float):
        self.threshold = threshold
        self.reset()

    def reset(self):
        self.cuts, self._cut, self._waiting, self._hw = [], set(), [], None

    def push(self, j: int, prev_u8: torch.Tensor, cur_u8: torch.Tensor):
        self._waiting.append((j, _pair_sums(prev_u8, cur_u8)))
        self._hw = tuple(cur_u8.shape[:2])

    def resolve(self):
        if not self._waiting:
            return
        scores = scores_from_sums(torch.cat([s for _, s in self._waiting], 0).cpu(), *self._hw).tolist()
        for (j, _), s in zip(self._waiting, scores):
            if s >= self.threshold:
                self.cuts.append(j)
                self._cut.add(j)
        self._waiting = []

    def __contains__(self, j: int) -> bool:
        return j in self._cut


def _as_output(u8: torch.Tensor, bgr: bool) -> torch.Tensor:
    """an input frame as an output frame: its bytes, BGR-flipped when `bgr`"""
    return u8.flip(-1) if bgr else u8.clone()


def flow_images(padder: InputPadder, flowt: List[torch.Tensor], bgr: bool) -> List[torch.Tensor]:
    """video_Nx.py:183-189: each (2,Hc,Wc) flowt cropped with the frames' padder (InputPadder.unpad_box) -> flow_to_image, one
    maximum per picture, computed on the GPU; the crop is read in place"""
    from .flow_viz import flow_to_image

    out = []
    for f in flowt:
        top, bottom, left, right = padder.unpad_box(f.shape[-2], f.shape[-1])
        out.append(flow_to_image(f.permute(1, 2, 0)[top:bottom, left:right], convert_to_bgr=bgr))
    return out


@torch.no_grad()
def interpolate_pair_u8(model, frame0_u8: torch.Tensor, frame1_u8: torch.Tensor, N: int = 2, ds_factor: Optional[float] = None,
                        bgr: bool = True, with_flow: bool = False):
    """One iteration of video_Nx.py's frame loop (:134-202): two (h,w,3) uint8 RGB frames -> the N-1 interpolated
    (h,w,3) uint8 frames at t = i/N.  with_flow: returns (frames, flow_images), the second being the N-1 colour-wheel pictures
    of the motion flowt (video_Nx.py:183-189, BGR when `bgr`), uint8 (h',w',3) on the device; only flowt is requested from the
    model besides the frames."""
    dev = frame0_u8.device
    padder = InputPadder(frame0_u8.shape[:2], 32)
    x = padder.pad_u8(torch.stack([frame0_u8, frame1_u8], 0))          # (2,3,H,W)
    xs = torch.stack([x[0], x[1]], 1).unsqueeze(0).contiguous()          # (1,3,2,H,W)
    H, W = xs.shape[-2:]
    ratio = 1.0 if ds_factor is None else ds_factor
    coords = [(model.sample_coord_input(1, (H, W), [i / N], device=dev, upsample_ratio=ratio), None) for i in range(1, N)]
    ts = [i / N * torch.ones(1, device=dev) for i in range(1, N)]
    out = model._interpolate(xs, coords, ts, ds_factor, ("flowt",) if with_flow else False)
    frames = [padder.unpad_u8(im, bgr)[0] for im in out["imgt_pred"]]
    return (frames, flow_images(padder, out["flowt"], bgr)) if with_flow else frames


class VideoInterpolator:
    """video_Nx.py's frame loop (src/video_Nx.py:134-216) as a streaming object: push() the frames of a clip one by one and
    get the N-1 interpolated frames between the previous frame and the new one.  Consecutive pairs share a frame, so the
    RAFT encoder products of each pair's second frame (fnet map, cnet net/inp, projected context features) stay in a device
    cache and are not recomputed when that frame becomes the next pair's first frame (SURVEY.md 8(f) row 2); the outputs
    are bit-identical to independent per-pair calls.  with_flow: push() returns (frames, flow_images) as
    interpolate_pair_u8(..., with_flow=True) does.

    pairs_per_call K > 1: push() buffers frames until K pairs are waiting, then interpolates them in one model.interpolate call
    (K + 1 frames, each encoded once; the last is kept as the next call's first frame) and returns the K (N-1) frames in clip order,
    pair by pair; the pushes in between return nothing.  flush() interpolates the pairs still waiting at the end of a clip.  With K = 1
    every push runs its pair at once, through the frame cache above.

    scene_threshold T (None: off): a pair of consecutive input frames whose scene_scores score is >= T is a hard cut and is not
    interpolated.  Its N - 1 frames at t = i / N are the nearer input frame, the earlier one for t <= 1/2 (its bytes, BGR-flipped when
    `bgr`), and with_flow gives the colour-wheel picture of a zero flow for each.  The score of a pair is computed on the device when its
    second frame is pushed and read back once per engine call (K = 1: once per push; K > 1: once per block of K pairs, of which only the
    pairs that are not cuts go to the engine, and none at all when every pair is one).  `cuts` lists the input indices j whose pair
    (j - 1, j) was a cut since the last reset().  With K = 1 the pair after a cut runs without the frame cache, which holds nothing of
    its first frame."""

    def __init__(self, model, N: int = 2, ds_factor: Optional[float] = None, bgr: bool = True, with_flow: bool = False,
                 pairs_per_call: int = 1, scene_threshold: Optional[float] = None):
        if int(pairs_per_call) < 1:
            raise ValueError("pairs_per_call must be >= 1, got %r" % (pairs_per_call,))
        self.scene_threshold = _scene_threshold(scene_threshold)
        self.model, self.N, self.ds, self.bgr, self.with_flow = model, int(N), ds_factor, bgr, bool(with_flow)
        self.pairs_per_call = int(pairs_per_call)
        self._prev = None      # padded float frame (3,H,W) of the last push
        self._padder = None
        self._cache = None     # uint8 device buffer holding the previous frame's encoder products
        self._cache_valid = False
        self._pending = []     # pairs_per_call > 1: the padded frames pushed after _prev, not yet interpolated
        self._scene = None if self.scene_threshold is None else _Cuts(self.scene_threshold)
        self._n = 0            # frames pushed since the last reset
        self._u8 = []          # scene detection: copies of the uint8 frames of _prev and _pending

    @property
    def cuts(self) -> List[int]:
        return list(self._scene.cuts) if self._scene is not None else []

    def reset(self):
        self._prev, self._cache_valid, self._pending = None, False, []
        self._n, self._u8 = 0, []
        if self._scene is not None:
            self._scene.reset()

    def _empty(self):
        return ([], []) if self.with_flow else []

    def _cut_frames(self, a_u8: torch.Tensor, b_u8: torch.Tensor):
        """the N - 1 outputs of a cut pair: the nearer input frame at each t = i / N (ties to the earlier), and zero-flow pictures"""
        N = self.N
        frames = [_as_output(a_u8 if 2 * i <= N else b_u8, self.bgr) for i in range(1, N)]
        if not self.with_flow:
            return frames, []
        H, W = self._padder.padded_shape
        ratio = 1.0 if self.ds is None else self.ds
        zero = torch.zeros(2, int(H * ratio), int(W * ratio), dtype=torch.float32, device=a_u8.device)
        return frames, flow_images(self._padder, [zero] * (N - 1), self.bgr)

    @torch.no_grad()
    def flush(self):
        """interpolate the pairs still buffered (pairs_per_call > 1) and return their frames as push() does; nothing is left waiting"""
        if not self._pending:
            return self._empty()
        k = len(self._pending)
        cut = [False] * k
        if self._scene is not None:
            self._scene.resolve()
            cut = [self._n - k + p in self._scene for p in range(k)]   # pair p is (input n - k + p - 1, n - k + p)
        keep = [p for p in range(k) if not cut[p]]
        N, aux = self.N, ("flowt",) if self.with_flow else False
        frames_u8, flows = [], []
        if keep:
            # only the frames of the pairs that are sent: with no cut, every frame and the pairs (i, i + 1)
            clip = [self._prev] + self._pending
            used = sorted({f for p in keep for f in (p, p + 1)})
            local = {f: i for i, f in enumerate(used)}
            frames = torch.stack([clip[f] for f in used], 0)               # (k+1,3,H,W) without a cut
            kk = len(keep)
            out = self.model._interpolate_clip(frames, [(local[p], local[p + 1]) for p in keep], [i / N for i in range(1, N)], self.ds, aux)
            # out["imgt_pred"][i] is (kk,3,H,W): timestep i of every pair -> clip order, pair by pair
            ims = torch.stack(out["imgt_pred"], 1).reshape(kk * (N - 1), *out["imgt_pred"][0].shape[1:])
            frames_u8 = list(self._padder.unpad_u8(ims, self.bgr).unbind(0)) if N > 1 else []
            if self.with_flow:
                fl = out["flowt"]   # T x (kk,2,Hc,Wc), or (2,Hc,Wc) when kk == 1 (forward's .squeeze())
                fl = [f.reshape(kk, *f.shape[-3:]) for f in fl]
                flows = flow_images(self._padder, [fl[i][p] for p in range(kk) for i in range(N - 1)], self.bgr)
        self._prev, self._pending = self._pending[-1], []
        if len(keep) < k:   # the cut pairs' frames in their places
            got_f, got_fl, frames_u8, flows = iter(frames_u8), iter(flows), [], []
            for p in range(k):
                if cut[p]:
                    f, fl = self._cut_frames(self._u8[p], self._u8[p + 1])
                else:
                    f = [next(got_f) for _ in range(N - 1)]
                    fl = [next(got_fl) for _ in range(N - 1)] if self.with_flow else []
                frames_u8 += f
                flows += fl
        if self._scene is not None:
            self._u8 = self._u8[-1:]
        return (frames_u8, flows) if self.with_flow else frames_u8

    @torch.no_grad()
    def push(self, frame_u8: torch.Tensor):
        dev = frame_u8.device
        if self._padder is None or (self._padder.ht, self._padder.wd) != tuple(frame_u8.shape[:2]):
            if self._pending:
                raise ValueError("VideoInterpolator: the frame size changed with pairs still buffered; flush() first")
            self._padder = InputPadder(frame_u8.shape[:2], 32)
            self.reset()
        cur = self._padder.pad_u8(frame_u8.unsqueeze(0))[0]              # (3,H,W)
        j = self._n
        self._n += 1
        if self._scene is not None:
            u8 = frame_u8.clone()   # the caller may reuse its buffer; a cut pair's outputs are these bytes
            if self._u8:
                self._scene.push(j, self._u8[-1], u8)
            self._u8.append(u8)
        if self._prev is None:
            self._prev = cur
            return self._empty()
        if self.pairs_per_call > 1:
            self._pending.append(cur)
            return self.flush() if len(self._pending) == self.pairs_per_call else self._empty()
        if self._scene is not None:
            self._scene.resolve()
            prev_u8, self._u8 = self._u8[0], self._u8[-1:]
            if j in self._scene:
                self._prev, self._cache_valid = cur, False   # the cache holds frame j - 1's products, not frame j's
                frames, flows = self._cut_frames(prev_u8, self._u8[0])
                return (frames, flows) if self.with_flow else frames
        m = self.model
        xs = torch.stack([self._prev, cur], 1).unsqueeze(0).contiguous()  # (1,3,2,H,W)
        H, W = xs.shape[-2:]
        ratio = 1.0 if self.ds is None else self.ds
        N = self.N
        coords = [(m.sample_coord_input(1, (H, W), [i / N], device=dev, upsample_ratio=ratio), None) for i in range(1, N)]
        ts = [i / N * torch.ones(1, device=dev) for i in range(1, N)]
        Hc, Wc = coords[0][0].shape[2:4]
        need = m.engine.frame_cache_bytes(1, H, W, N - 1, self.ds, Hc, Wc)
        if self._cache is None or self._cache.numel() < need or self._cache.device != dev:
            self._cache, self._cache_valid = torch.empty(need, dtype=torch.uint8, device=dev), False
        aux = ("flowt",) if self.with_flow else False
        # The engine keeps its own record of what each cache buffer holds (problem size, precision mode; cleared when the weights
        # change): a refused load -> one full forward with load=False.  The signature adds what only the caller can know.
        sig = (id(m.engine), int(m.tensor_cores), m.engine.weights_version)
        load = self._cache_valid and getattr(self, "_cache_sig", None) == sig
        try:
            try:
                out = m._interpolate(xs, coords, ts, self.ds, aux, frame_cache=(self._cache, load, True))
            except GimmvfiError as ex:
                if not (load and "frame cache" in str(ex)):
                    raise
                out = m._interpolate(xs, coords, ts, self.ds, aux, frame_cache=(self._cache, False, True))
            self._cache_valid, self._cache_sig = True, sig
        except Exception:
            self._cache_valid = False
            raise
        self._prev = cur
        frames = [self._padder.unpad_u8(im, self.bgr)[0] for im in out["imgt_pred"]]
        return (frames, flow_images(self._padder, out["flowt"], self.bgr)) if self.with_flow else frames


def _rate(x, name: str) -> Fraction:
    """a frame rate as an exact rational: an int, a Fraction, or a string such as "30000/1001" or "29.97" (floats via their repr)"""
    if isinstance(x, bool) or not isinstance(x, (int, float, str, Fraction)):
        raise ValueError("%s must be an int, a Fraction or a string such as '30000/1001', got %r" % (name, x))
    try:
        r = Fraction(repr(x) if isinstance(x, float) else x.strip() if isinstance(x, str) else x)
    except (ValueError, ZeroDivisionError):
        raise ValueError("%s: cannot read %r as a frame rate" % (name, x))
    if r <= 0:
        raise ValueError("%s must be positive, got %s" % (name, r))
    return r


SNAP = Fraction(1, 10 ** 6)   # output instants this close to an input frame (in input frames) are that frame


class FrameRateConverter:
    """Frame-rate conversion of a clip streamed frame by frame: push() the (h,w,3) uint8 RGB input frames, get the output frames at
    fps_out.  Output frame k shows input time tau_k = k * fps_in / fps_out (in input frames, exact rationals: no drift), for every k with
    tau_k <= the last input frame.  A tau_k within SNAP (1e-6 input frames) of an input frame is that frame itself (no engine work; its
    bytes, BGR-flipped when `bgr`); any other is the query (floor(tau), floor(tau) + 1, float32(tau - floor(tau))) of
    GIMMVFI_R / GIMMVFI_F.interpolate_at, whose t then lies strictly inside (0, 1).  The tolerance matters for rates given as decimal
    approximations, e.g. 30000/1001 as the float 29.97002997002997 that video readers report: their instants land a hair off the
    input frames, where float32(t) rounds to 0 or 1 or the lookup's 1/t scaling is ill-conditioned; and no picture a hair away from
    an input frame differs from it.  The converter keeps its own copy of the last frame pushed, so a caller may reuse its buffer.
    Up to pairs_per_call K pairs that have queries go into one call, each frame encoded once; pairs without a query (60 -> 24 has
    them) are never sent, and equal rates make no engine call at all.  Frames come back in output order: push() returns those that are
    complete, flush() the rest at the end of a clip.  Pre- and post-processing are VideoInterpolator's (InputPadder, GPU uint8).
    A call's workspace grows with K (model.engine.queries_workspace_bytes): at 1080p GIMM-VFI-R fits K = 4 for 24 -> 60 on an 80 GB
    device but only K = 1 for 60 -> 24, whose pairs do not share frames (DESIGN §7).

    scene_threshold T (None: off): a pair of consecutive input frames whose scene_scores score is >= T is a hard cut and is never sent to
    the engine.  An output instant at offset t into a cut interval is the nearer input frame, the earlier one for t <= 1/2 (its bytes,
    BGR-flipped when `bgr`).  The score of (j - 1, j) is computed on the device when frame j is pushed; the scores are read back once per
    engine call or flush(), when the K pairs with queries of a call are decided, and a call whose pairs are all cuts is not made.
    `cuts` lists the input indices j whose pair (j - 1, j) scored >= T since the last reset()."""

    def __init__(self, model, fps_in, fps_out, ds_factor: Optional[float] = None, bgr: bool = True, pairs_per_call: int = 1,
                 scene_threshold: Optional[float] = None):
        if isinstance(pairs_per_call, bool) or int(pairs_per_call) < 1:
            raise ValueError("pairs_per_call must be >= 1, got %r" % (pairs_per_call,))
        self.scene_threshold = _scene_threshold(scene_threshold)
        self.model, self.ds, self.bgr, self.pairs_per_call = model, ds_factor, bgr, int(pairs_per_call)
        self.fps_in, self.fps_out = _rate(fps_in, "fps_in"), _rate(fps_out, "fps_out")
        self.step = self.fps_in / self.fps_out   # input frames per output frame
        self._padder = None
        self._scene = None if self.scene_threshold is None else _Cuts(self.scene_threshold)
        self.reset()

    @property
    def cuts(self) -> List[int]:
        return list(self._scene.cuts) if self._scene is not None else []

    def reset(self):
        """start a new clip: the next frame pushed is input frame 0"""
        self._n = 0             # input frames pushed
        self._k = 0             # next output index to schedule
        self._prev_u8 = None    # a copy of the last frame pushed
        # scheduled outputs, in order: ("frame", uint8 (h,w,3)) or ("query", src, tgt, t, the input frame shown if (src, tgt) is a cut)
        self._queue = []
        self._frames = {}       # input index -> padded float frame (3,H,W), for the queries waiting
        if self._scene is not None:
            self._scene.reset()

    @torch.no_grad()
    def flush(self) -> List[torch.Tensor]:
        """interpolate the queries waiting and return every scheduled output frame, in order"""
        return self._emit(True)

    def _emit(self, decide: bool) -> List[torch.Tensor]:
        """flush(); decide: read the waiting scene scores first (push() skips it when no query waits)"""
        if decide and self._scene is not None:
            self._scene.resolve()
            self._queue = [("frame", _as_output(e[4], self.bgr)) if e[0] == "query" and e[2] in self._scene else e for e in self._queue]
        queries = [e[1:4] for e in self._queue if e[0] == "query"]
        preds = iter(())
        if queries:
            used = sorted({f for a, b, _ in queries for f in (a, b)})   # without a cut: every frame in self._frames
            local = {f: i for i, f in enumerate(used)}
            frames = torch.stack([self._frames[f] for f in used], 0)
            out = self.model._interpolate_at(frames, [(local[a], local[b], t) for a, b, t in queries], self.ds, False)
            preds = iter(self._padder.unpad_u8(out["imgt_pred"], self.bgr).unbind(0))
        res = [e[1] if e[0] == "frame" else next(preds) for e in self._queue]
        self._queue, self._frames = [], {}
        return res

    @torch.no_grad()
    def push(self, frame_u8: torch.Tensor) -> List[torch.Tensor]:
        """the next input frame, (h,w,3) uint8 RGB -> the output frames completed by it, in order (uint8 (h,w,3), BGR when `bgr`)"""
        if self._padder is None or (self._padder.ht, self._padder.wd) != tuple(frame_u8.shape[:2]):
            if self._queue:
                raise ValueError("FrameRateConverter: the frame size changed with frames still waiting; flush() first")
            self._padder = InputPadder(frame_u8.shape[:2], 32)
            self.reset()
        j = self._n
        self._n += 1
        cur_u8 = frame_u8.clone()
        if self._scene is not None and j > 0:
            self._scene.push(j, self._prev_u8, cur_u8)
        while self._k * self.step <= j:   # the output instants in (j - 1, j] (frame 0: the instant 0)
            off = self._k * self.step - (j - 1)   # in (0, 1]
            self._k += 1
            if off >= 1 - SNAP or off <= SNAP:    # input frame j, or (a hair after it) frame j - 1
                self._queue.append(("frame", _as_output(cur_u8 if off >= 1 - SNAP else self._prev_u8, self.bgr)))
                continue
            for f, u8 in ((j - 1, self._prev_u8), (j, cur_u8)):
                if f not in self._frames:
                    self._frames[f] = self._padder.pad_u8(u8.unsqueeze(0))[0]
            near = self._prev_u8 if off <= Fraction(1, 2) else cur_u8   # the output if (j - 1, j) is a cut
            self._queue.append(("query", j - 1, j, float(np.float32(float(off))), near))
        self._prev_u8 = cur_u8
        waiting = {(e[1], e[2]) for e in self._queue if e[0] == "query"}
        if not waiting:
            return self._emit(False)
        return self._emit(True) if len(waiting) >= self.pairs_per_call else []
