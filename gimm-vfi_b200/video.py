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


def _forward_pair(model, x0: torch.Tensor, x1: torch.Tensor, N: int, ds_factor: Optional[float], aux, frame_cache=None):
    """model._interpolate on one pair of padded (3,H,W) frames at t = i/N, i = 1 .. N-1, the coordinates sample_coord_input's at
    ds_factor.  frame_cache: None, or (buffer, load, store) as EngineHandle.forward takes it.  The engine keeps its own record of what a
    buffer holds (problem size, precision mode; cleared when the weights change), and a load it refuses is retried once as a full
    forward with load=False."""
    dev = x0.device
    xs = torch.stack([x0, x1], 1).unsqueeze(0).contiguous()          # (1,3,2,H,W)
    H, W = xs.shape[-2:]
    ratio = 1.0 if ds_factor is None else ds_factor
    coords = [(model.sample_coord_input(1, (H, W), [i / N], device=dev, upsample_ratio=ratio), None) for i in range(1, N)]
    ts = [i / N * torch.ones(1, device=dev) for i in range(1, N)]
    try:
        return model._interpolate(xs, coords, ts, ds_factor, aux, frame_cache=frame_cache)
    except GimmvfiError as ex:
        if not (frame_cache is not None and frame_cache[1] and "frame cache" in str(ex)):
            raise
        return model._interpolate(xs, coords, ts, ds_factor, aux, frame_cache=(frame_cache[0], False, frame_cache[2]))


@torch.no_grad()
def interpolate_pair_u8(model, frame0_u8: torch.Tensor, frame1_u8: torch.Tensor, N: int = 2, ds_factor: Optional[float] = None,
                        bgr: bool = True, with_flow: bool = False):
    """One iteration of video_Nx.py's frame loop (:134-202): two (h,w,3) uint8 RGB frames -> the N-1 interpolated
    (h,w,3) uint8 frames at t = i/N.  with_flow: returns (frames, flow_images), the second being the N-1 colour-wheel pictures
    of the motion flowt (video_Nx.py:183-189, BGR when `bgr`), uint8 (h',w',3) on the device; only flowt is requested from the
    model besides the frames."""
    padder = InputPadder(frame0_u8.shape[:2], 32)
    x = padder.pad_u8(torch.stack([frame0_u8, frame1_u8], 0))          # (2,3,H,W)
    out = _forward_pair(model, x[0], x[1], N, ds_factor, ("flowt",) if with_flow else False)
    frames = [padder.unpad_u8(im, bgr)[0] for im in out["imgt_pred"]]
    return (frames, flow_images(padder, out["flowt"], bgr)) if with_flow else frames


class _Stream:
    """What VideoInterpolator and FrameRateConverter share: a clip's input frames, pushed one by one, become a stream of outputs.  Pushing
    input frame j schedules the output instants in (j - 1, j] (the subclass's _instants).  An output is an input frame passed through, or
    the interpolation of the pair (j - 1, j) at some t, which falls back to the nearer input frame (offset <= 1/2: the earlier) if the
    pair turns out to be a scene cut.  The outputs wait in a queue in output order.  A push that leaves no interpolation waiting returns
    the queue and reads nothing back.  A push that brings the distinct pairs waiting to pairs_per_call, and flush(), read every waiting
    scene score in one copy, turn the entries of cut pairs into their fallback frames, and send the pairs left to one engine call (the
    subclass's _run) on only the frames they use; then the whole queue comes back in order."""

    with_flow = False
    _passes_frames = False   # whether an output instant can fall on an input frame (then uint8 copies are always kept)

    def __init__(self, model, ds_factor: Optional[float], bgr: bool, pairs_per_call: int, scene_threshold: Optional[float]):
        self.scene_threshold = _scene_threshold(scene_threshold)
        self.model, self.ds, self.bgr, self.pairs_per_call = model, ds_factor, bgr, int(pairs_per_call)
        self._padder = None
        self._scene = None if self.scene_threshold is None else _Cuts(self.scene_threshold)
        # uint8 copies of the input frames, kept only where an output can be one: a pass-through frame or a cut's fallback
        self._copies = self._passes_frames or self._scene is not None
        self.reset()

    @property
    def cuts(self) -> List[int]:
        return list(self._scene.cuts) if self._scene is not None else []

    def reset(self):
        """start a new clip: the next frame pushed is input frame 0"""
        self._n = 0             # input frames pushed
        # the scheduled outputs, in order: ((j - 1, j), t, fallback) for an interpolation, (None, None, frame) for an input frame, the
        # frames being our uint8 copies (None without copies)
        self._queue = []
        self._padded = {}       # input index -> padded float frame (3,H,W): the frames of the pairs waiting, and the last frame
        self._last_u8 = None    # the copy of the last frame pushed
        if self._scene is not None:
            self._scene.reset()

    def _net_size(self, H: int, W: int):
        """the network-resolution size of padded H x W frames: sample_coord_input's grid at ds_factor"""
        ratio = 1.0 if self.ds is None else self.ds
        return int(H * ratio), int(W * ratio)

    @torch.no_grad()
    def flush(self):
        """interpolate what is waiting and return every output scheduled, in order, as push() does; nothing is left waiting"""
        return self._emit(True)

    @torch.no_grad()
    def push(self, frame_u8: torch.Tensor):
        """the next input frame, (h,w,3) uint8 RGB on the device -> the outputs completed by it, in order (uint8 (h,w,3), BGR when `bgr`)"""
        if self._padder is None or (self._padder.ht, self._padder.wd) != tuple(frame_u8.shape[:2]):
            if self._queue:
                raise ValueError("%s: the frame size changed with outputs still waiting; flush() first" % type(self).__name__)
            self._padder = InputPadder(frame_u8.shape[:2], 32)
            self.reset()
        j = self._n
        self._n += 1
        prev_u8, cur_u8 = self._last_u8, (frame_u8.clone() if self._copies else None)   # the caller may reuse its buffer
        if self._scene is not None and j > 0:
            self._scene.push(j, prev_u8, cur_u8)
        if cur_u8 is None:   # the padded frame is then the only copy of frame j that the next pair can use
            self._padded[j] = self._padder.pad_u8(frame_u8.unsqueeze(0))[0]
        for off, t in self._instants(j):
            fallback = prev_u8 if off <= Fraction(1, 2) else cur_u8
            if t is None:
                self._queue.append((None, None, fallback))
                continue
            for f, u8 in ((j - 1, prev_u8), (j, frame_u8)):
                if f not in self._padded:
                    self._padded[f] = self._padder.pad_u8(u8.unsqueeze(0))[0]
            self._queue.append(((j - 1, j), t, fallback))
        self._last_u8 = cur_u8
        waiting = {pair for pair, _, _ in self._queue if pair is not None}
        if waiting and len(waiting) < self.pairs_per_call:
            return ([], []) if self.with_flow else []
        return self._emit(bool(waiting))

    def _emit(self, decide: bool):
        """every output in the queue, in order, leaving it empty.  decide: read the waiting scene scores first and turn the entries of
        cut pairs into their fallback frames.  An engine call that raises drops the outputs it was to make, and the clip goes on with the
        next frame pushed."""
        if decide and self._scene is not None:
            self._scene.resolve()
            self._queue = [(None, None, u8) if pair is not None and pair[1] in self._scene else (pair, t, u8) for pair, t, u8 in self._queue]
        queue, self._queue = self._queue, []
        interp = [(pair, t) for pair, t, _ in queue if pair is not None]
        preds = flows = iter(())
        if interp:
            used = sorted({f for pair, _ in interp for f in pair})   # without a cut: every frame since the last call
            local = {f: i for i, f in enumerate(used)}
            ims, fl = self._run(used, [self._padded[f] for f in used], [(local[a], local[b], t) for (a, b), t in interp])
            preds, flows = iter(self._padder.unpad_u8(ims, self.bgr).unbind(0)), iter(fl or ())
        self._padded = {f: x for f, x in self._padded.items() if f == self._n - 1}
        frames = [next(preds) if pair is not None else _as_output(u8, self.bgr) for pair, _, u8 in queue]
        if not self.with_flow:
            return frames
        zero = None
        if len(interp) < len(queue):   # a cut's pictures are those of a zero flow at the network resolution
            zero = torch.zeros(2, *self._net_size(*self._padder.padded_shape), dtype=torch.float32, device=queue[0][2].device)
        pics = [next(flows) if pair is not None else zero for pair, _, _ in queue]
        return frames, (flow_images(self._padder, pics, self.bgr) if pics else [])


class VideoInterpolator(_Stream):
    """video_Nx.py's frame loop (src/video_Nx.py:134-216) as a streaming object: push() the frames of a clip one by one and
    get the N-1 interpolated frames at t = i/N between the previous frame and the new one (N >= 2).  Consecutive pairs share a frame, so
    the RAFT encoder products of each pair's second frame (fnet map, cnet net/inp, projected context features) stay in a device cache
    and are not recomputed when that frame becomes the next pair's first frame (SURVEY.md 8(f) row 2); the outputs are bit-identical
    to independent per-pair calls.  A pair loads the cache only when it holds the pair's first frame, under the same engine, precision
    mode and weights.  with_flow: push() returns (frames, flow_images) as interpolate_pair_u8(..., with_flow=True) does.

    pairs_per_call K > 1: push() buffers frames until K pairs are waiting, then interpolates them in one model.interpolate call
    (K + 1 frames, each encoded once; the last is kept as the next call's first frame) and returns the K (N-1) frames in clip order,
    pair by pair; the pushes in between return nothing.  flush() interpolates the pairs still waiting at the end of a clip.  With K = 1
    every push runs its pair at once, through the frame cache above.

    scene_threshold T (None: off): a pair of consecutive input frames whose scene_scores score is >= T is a hard cut and is not
    interpolated.  Its N - 1 frames at t = i / N are the nearer input frame, the earlier one for t <= 1/2 (its bytes, BGR-flipped when
    `bgr`), and with_flow gives the colour-wheel picture of a zero flow for each.  The score of a pair is computed on the device when its
    second frame is pushed and read back once per engine call (K = 1: once per push; K > 1: once per block of K pairs, of which only the
    pairs that are not cuts go to the engine, and none at all when every pair is one).  `cuts` lists the input indices j whose pair
    (j - 1, j) was a cut since the last reset().  With K = 1 the pair after a cut does not load the frame cache, which holds the products
    of the frame before the cut."""

    def __init__(self, model, N: int = 2, ds_factor: Optional[float] = None, bgr: bool = True, with_flow: bool = False,
                 pairs_per_call: int = 1, scene_threshold: Optional[float] = None):
        if int(pairs_per_call) < 1:
            raise ValueError("pairs_per_call must be >= 1, got %r" % (pairs_per_call,))
        if int(N) < 2:
            raise ValueError("N must be >= 2 (the N - 1 frames between two input frames are at t = i / N), got %r" % (N,))
        self.N, self.with_flow = int(N), bool(with_flow)
        self._cache = None     # uint8 device buffer holding the encoder products of the frame self._cached names
        super().__init__(model, ds_factor, bgr, pairs_per_call, scene_threshold)

    def reset(self):
        super().reset()
        self._cached = None    # (input index of the frame whose products the frame cache holds, signature), or None

    def _instants(self, j: int):
        return [(Fraction(i, self.N), i / self.N) for i in range(1, self.N)] if j > 0 else []

    def _run(self, used, frames, queries):
        """one engine call on the waiting pairs -> their predictions (n,3,H,W) and with_flow their flowt, in queue order"""
        N, aux = self.N, ("flowt",) if self.with_flow else False
        pairs = list(dict.fromkeys((a, b) for a, b, _ in queries))
        if self.pairs_per_call > 1:
            out = self.model._interpolate_clip(torch.stack(frames, 0), pairs, [i / N for i in range(1, N)], self.ds, aux)
        else:
            out = self._forward_cached(used, frames, aux)
        # out[key][i] holds timestep i of every pair -> queue order, pair by pair
        P = len(pairs)
        ims = torch.stack(out["imgt_pred"], 1).reshape(P * (N - 1), *out["imgt_pred"][0].shape[1:])
        if not self.with_flow:
            return ims, None
        fl = [f.reshape(P, *f.shape[-3:]) for f in out["flowt"]]   # (2,Hc,Wc) for a single pair (forward's .squeeze())
        return ims, [fl[i][p] for p in range(P) for i in range(N - 1)]

    def _forward_cached(self, used, frames, aux):
        """pairs_per_call 1: the pair's forward through the frame cache, loading it when it holds the pair's first frame"""
        m, (a, b), dev = self.model, used, frames[0].device
        H, W = frames[0].shape[-2:]
        need = m.engine.frame_cache_bytes(1, H, W, self.N - 1, self.ds, *self._net_size(H, W))
        if self._cache is None or self._cache.numel() < need or self._cache.device != dev:
            self._cache, self._cached = torch.empty(need, dtype=torch.uint8, device=dev), None
        # the engine refuses a load its own record of the buffer does not match; the signature adds what only the caller can know
        sig = (id(m.engine), int(m.tensor_cores), m.engine.weights_version)
        held, self._cached = self._cached, None   # after an exception, the cache holds nothing known
        out = _forward_pair(m, frames[0], frames[1], self.N, self.ds, aux, frame_cache=(self._cache, held == (a, sig), True))
        self._cached = (b, sig)
        return out


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


class FrameRateConverter(_Stream):
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

    _passes_frames = True

    def __init__(self, model, fps_in, fps_out, ds_factor: Optional[float] = None, bgr: bool = True, pairs_per_call: int = 1,
                 scene_threshold: Optional[float] = None):
        if isinstance(pairs_per_call, bool) or int(pairs_per_call) < 1:
            raise ValueError("pairs_per_call must be >= 1, got %r" % (pairs_per_call,))
        super().__init__(model, ds_factor, bgr, pairs_per_call, scene_threshold)
        self.fps_in, self.fps_out = _rate(fps_in, "fps_in"), _rate(fps_out, "fps_out")
        self.step = self.fps_in / self.fps_out   # input frames per output frame

    def reset(self):
        super().reset()
        self._k = 0             # next output index to schedule

    def _instants(self, j: int):
        while self._k * self.step <= j:   # the output instants in (j - 1, j] (frame 0: the instant 0)
            off = self._k * self.step - (j - 1)   # in (0, 1]
            self._k += 1
            # input frame j, or (a hair after it) frame j - 1; any other instant is interpolated at the float32 t the engine receives
            yield off, None if off >= 1 - SNAP or off <= SNAP else float(np.float32(float(off)))

    def _run(self, used, frames, queries):
        return self.model._interpolate_at(torch.stack(frames, 0), queries, self.ds, False)["imgt_pred"], None
