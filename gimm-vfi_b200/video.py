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
        self.decided = 0   # every pair (j - 1, j) with j <= decided has been read back

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
        self.decided = self._waiting[-1][0]
        self._waiting = []

    def __contains__(self, j: int) -> bool:
        return j in self._cut


def _as_output(u8: torch.Tensor, bgr: bool) -> torch.Tensor:
    """an input frame as an output frame: its bytes, BGR-flipped when `bgr`"""
    return u8.flip(-1) if bgr else u8.clone()


def blend_u8(sources: List[torch.Tensor], padder: InputPadder, bgr: bool = True) -> torch.Tensor:
    """gimmvfi_op_blend_u8: one (h,w,3) uint8 output frame as the mean of 1 to 63 sources on one device, each a padded (3,H,W) float32
    engine prediction (value x * 255, cropped with the padder's unpad box) or an (h,w,3) uint8 RGB frame (value its byte), both
    contiguous.  Each channel is the float32 sum over the sources in order, then trunc(clamp(sum / n, 0, 255)): one source gives
    unpad_u8's bytes, and n copies of one frame give that frame.  BGR when `bgr`.  One launch."""
    n = len(sources)
    if not 1 <= n <= 63:
        raise ValueError("blend_u8: 1 to 63 sources, got %d" % n)
    h, w = padder.ht, padder.wd
    H, W = padder.padded_shape
    top, _, left, _ = padder.unpad_box(H, W)
    dev = sources[0].device
    for s in sources:
        shape = (3, H, W) if s.dtype == torch.float32 else (h, w, 3)
        if s.dtype not in (torch.float32, torch.uint8) or tuple(s.shape) != shape or not s.is_contiguous() or s.device != dev:
            raise ValueError("blend_u8: a source must be a contiguous (3,%d,%d) float32 or (%d,%d,3) uint8 tensor on %s, got %s %s"
                             % (H, W, h, w, dev, tuple(s.shape), s.dtype))
    out = torch.empty(h, w, 3, dtype=torch.uint8, device=dev)
    ptrs = (C.c_void_p * n)(*[s.data_ptr() for s in sources])
    kinds = (C.c_int * n)(*[int(s.dtype == torch.float32) for s in sources])
    lib = default_lib()
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream) if dev.type == "cuda" else None
    lib.check(lib.dll.gimmvfi_op_blend_u8(ptrs, kinds, n, H, W, top, left, C.c_void_p(out.data_ptr()), h, w, int(bgr), stream))
    return out


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


class _Sample:
    """one instant of an output: input frame f (u8: our uint8 copy of it, None without copies), or the interpolation of pair (j - 1, j) at
    t, which falls back to frame f, the nearer one (offset <= 1/2: the earlier), if the pair turns out to be a scene cut.  After the engine
    call, `out` holds what it made of the instant (the output frame, or with a shutter the padded float prediction) and `flow` its flowt."""

    __slots__ = ("pair", "t", "f", "u8", "out", "flow")

    def __init__(self, pair, t, f: int, u8: Optional[torch.Tensor]):
        self.pair, self.t, self.f, self.u8, self.out, self.flow = pair, t, f, u8, None, None


class _Entry:
    """one output frame in the queue: its samples in time order, `own` the one at the output's own instant.  Only a shutter's outputs
    have more than one sample: `pending` holds the instants of the window not placed yet (after the last frame pushed), `needs` the last
    j whose pair (j - 1, j) must be decided (scene score read back) before the output's shot is known, `tau` its own instant."""

    __slots__ = ("samples", "own", "pending", "needs", "tau")

    def __init__(self, samples=(), pending=(), needs: int = 0, tau=None):
        self.samples, self.pending, self.needs, self.tau = list(samples), list(pending), needs, tau
        self.own = self.samples[0] if len(self.samples) == 1 else None


class _Stream:
    """What VideoInterpolator and FrameRateConverter share: a clip's input frames, pushed one by one, become a stream of outputs.  An
    output is a queue entry holding one sample, or with FrameRateConverter's shutter the samples of its exposure window.  Pushing input
    frame j places the instants in (j - 1, j] (the subclass's _schedule): a sample is an input frame passed through, or the interpolation
    of the pair (j - 1, j) at some t, which falls back to the nearer input frame (offset <= 1/2: the earlier) if the pair turns out to be a
    scene cut.  The outputs wait in a queue in output order.  A push that leaves no interpolation waiting returns the complete outputs at
    the head of the queue and reads nothing back, unless the head waits only for scene scores (a shutter window of input frames alone):
    then it reads them back in one copy.  A push that brings the distinct pairs waiting to pairs_per_call, and flush(), read every
    waiting scene score in one copy, turn the samples of cut pairs into their fallback frames, and send the pairs left to one engine call
    (the subclass's _run) on only the frames they use; then the complete outputs come back in order.  An output is complete when each of
    its samples is placed and made, and the pairs its window spans are decided; without a shutter that is every output after a call.  An
    output still waiting after a call keeps copies of its sub-frames, so what waits is at most a few frames per output."""

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
        self._queue = []        # the scheduled outputs (_Entry), in order
        self._padded = {}       # input index -> padded float frame (3,H,W): the frames of the pairs waiting, and the last frame
        self._last_u8 = None    # the copy of the last frame pushed
        self._ended = False     # flush() ended the clip: the next push starts a new one
        if self._scene is not None:
            self._scene.reset()

    def _net_size(self, H: int, W: int):
        """the network-resolution size of padded H x W frames: sample_coord_input's grid at ds_factor"""
        ratio = 1.0 if self.ds is None else self.ds
        return int(H * ratio), int(W * ratio)

    @torch.no_grad()
    def flush(self):
        """interpolate what is waiting and return every output scheduled, in order, as push() does; nothing is left waiting"""
        return self._emit(True, final=True)

    @torch.no_grad()
    def push(self, frame_u8: torch.Tensor):
        """the next input frame, (h,w,3) uint8 RGB on the device -> the outputs completed by it, in order (uint8 (h,w,3), BGR when `bgr`)"""
        if self._ended:
            self.reset()
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
        self._schedule(j, prev_u8, frame_u8, cur_u8)
        self._last_u8 = cur_u8
        waiting = {s.pair for e in self._queue for s in e.samples if s.pair is not None and s.out is None}
        if waiting and len(waiting) < self.pairs_per_call:
            return ([], []) if self.with_flow else []
        # an output whose samples are all placed and made may still wait for the scores of the pairs its window spans (a shutter whose
        # samples all fall on input frames makes no engine call): read them back now rather than at the next call
        head = self._queue[0] if self._queue else None
        blocked = self._scene is not None and head is not None and not head.pending and head.needs > self._scene.decided
        return self._emit(bool(waiting) or blocked)

    def _schedule(self, j: int, prev_u8, frame_u8, cur_u8):
        """queue one output per instant of the subclass's _instants(j)"""
        for off, t in self._instants(j):
            self._queue.append(_Entry([self._sample(j, off, t, prev_u8, frame_u8, cur_u8)]))

    def _sample(self, j: int, off: Fraction, t: Optional[float], prev_u8, frame_u8, cur_u8) -> _Sample:
        """the sample at offset off in (0, 1] into (j - 1, j]: an input frame when t is None, else the query (j - 1, j, t)"""
        f, u8 = (j - 1, prev_u8) if off <= Fraction(1, 2) else (j, cur_u8)
        if t is None:
            return _Sample(None, None, f, u8)
        for g, x in ((j - 1, prev_u8), (j, frame_u8)):
            if g not in self._padded:
                self._padded[g] = self._padder.pad_u8(x.unsqueeze(0))[0]
        return _Sample((j - 1, j), t, f, u8)

    def _emit(self, decide: bool, final: bool = False):
        """the complete outputs at the head of the queue, in order (final: every output).  decide: read the waiting scene scores first and
        turn the samples of cut pairs into their fallback frames.  An engine call that raises drops the outputs waiting, and the clip goes
        on with the next frame pushed."""
        if decide and self._scene is not None:
            self._scene.resolve()
            for e in self._queue:
                for s in e.samples:
                    if s.pair is not None and s.pair[1] in self._scene:
                        s.pair = s.t = None
        if final:
            self._end_clip()
        queue, self._queue = self._queue, []
        interp = [s for e in queue for s in e.samples if s.pair is not None and s.out is None]
        if interp:
            used = sorted({f for s in interp for f in s.pair})   # without a cut: every frame since the last call
            local = {f: i for i, f in enumerate(used)}
            ims, fl = self._run(used, [self._padded[f] for f in used], [(local[s.pair[0]], local[s.pair[1]], s.t) for s in interp])
            for s, x in zip(interp, self._preds(ims)):
                s.out = x
            for s, x in zip(interp, fl or ()):
                s.flow = x
        self._padded = {f: x for f, x in self._padded.items() if f == self._n - 1}
        decided = self._n - 1 if self._scene is None else self._scene.decided
        n = len(queue) if final else next((i for i, e in enumerate(queue) if e.pending or e.needs > decided), len(queue))
        done, self._queue = queue[:n], queue[n:]
        made = set(interp)
        for e in self._queue:   # an output still waiting keeps copies of its sub-frames, not the whole output of this call
            for s in e.samples:
                if s in made:
                    s.out = s.out.clone()
        frames = [self._output(e) for e in done]
        if not self.with_flow:
            return frames
        zero = None
        if len(interp) < len(done):   # a cut's pictures are those of a zero flow at the network resolution
            zero = torch.zeros(2, *self._net_size(*self._padder.padded_shape), dtype=torch.float32, device=done[0].own.u8.device)
        pics = [e.own.flow if e.own.flow is not None else zero for e in done]
        return frames, (flow_images(self._padder, pics, self.bgr) if pics else [])

    def _end_clip(self):
        """flush(): the last input frame is known"""

    def _preds(self, ims: torch.Tensor):
        """the engine's predictions (n,3,H,W), in sample order -> what the samples keep: here their uint8 output frames"""
        return self._padder.unpad_u8(ims, self.bgr).unbind(0)

    def _output(self, e: _Entry) -> torch.Tensor:
        """a complete entry's output frame"""
        s = e.own
        return s.out if s.out is not None else _as_output(s.u8, self.bgr)


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


def _shutter_angle(x) -> Optional[Fraction]:
    """None, or a shutter angle in degrees in (0, 360] as an exact rational (floats via their repr, as _rate reads them)"""
    if x is None:
        return None
    if isinstance(x, bool) or not isinstance(x, numbers.Real):
        raise ValueError("shutter_angle must be None or a number in (0, 360], got %r" % (x,))
    try:
        a = Fraction(x) if isinstance(x, numbers.Rational) else Fraction(repr(float(x)))
    except (ValueError, OverflowError):
        raise ValueError("shutter_angle must be None or a number in (0, 360], got %r" % (x,))
    if not 0 < a <= 360:
        raise ValueError("shutter_angle must be None or a number in (0, 360], got %r" % (x,))
    return a


def _shutter_samples(x) -> int:
    if isinstance(x, bool) or not isinstance(x, numbers.Integral) or not 1 <= x <= 63 or x % 2 == 0:
        raise ValueError("shutter_samples must be an odd int in [1, 63], got %r" % (x,))
    return int(x)


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
    `cuts` lists the input indices j whose pair (j - 1, j) scored >= T since the last reset().

    shutter_angle A (None: off), shutter_samples S (odd, 1 .. 63; default 7): motion blur, as a camera whose shutter is open for A / 360 of
    each output frame.  Output k's exposure window is w = (A / 360) * fps_in / fps_out input frames wide, centred on tau_k, and its samples
    are the midpoints of S equal parts of it, s_i = tau_k - w / 2 + (i + 1/2) w / S (exact rationals).  A <= 360 keeps windows apart, so no
    two outputs share an instant.  Each sample takes the rule of an output instant above (an input frame within SNAP, a query, the nearer
    frame in a cut pair).  A sample before frame 0 or after the last frame is dropped, and so is one whose frame or pair lies in another
    shot than the output's own (a shot: the frames between two cuts).  The output's own shot is that of tau_k, the middle sample, which is
    why S is odd: that sample is never dropped, and it is the instant the converter shows without a shutter.  With an even S and a wide
    window every sample could land in another shot (120 -> 24 at 360 degrees with S = 2 around a one-frame shot).  The output is the mean of
    the n samples kept, each channel trunc(clamp(sum / n, 0, 255)) of the float32 sum in sample order of x * 255 (an engine frame) or the
    byte (an input frame): gimmvfi_op_blend_u8 (blend_u8), one launch per output frame.  S = 1 gives the bytes of shutter_angle=None for
    a clip ended by one flush(); unlike the converter without a shutter, a shutter's flush() always ends the clip (below).
    Averaging is in the frames' encoded values, as ffmpeg's tmix does; the window adds to the blur the input already has.  A pair still goes
    to exactly one engine call, with every sample any output places in it: pushing frame j places every sample in (j - 1, j], including
    those of outputs whose tau_k lies up to w / 2 after frame j, and an output comes back once each pair its window spans is decided and
    interpolated (the push that completes a window of input frames alone reads its scene scores back itself).  The sub-frames of an output are kept until it is complete, so its bytes do not depend on K.  flush() ends the clip:
    samples after the last frame are dropped, so the windows that cross the end are cut short and the clip cannot go on; the next push()
    starts a new clip (input frame 0, `cuts` cleared).  Without a shutter, flush() leaves the clip open, as it always has.  The samples of
    an output past the end of the clip (at most one output's) may have been interpolated by then and are thrown away."""

    _passes_frames = True

    def __init__(self, model, fps_in, fps_out, ds_factor: Optional[float] = None, bgr: bool = True, pairs_per_call: int = 1,
                 scene_threshold: Optional[float] = None, shutter_angle=None, shutter_samples: int = 7):
        if isinstance(pairs_per_call, bool) or int(pairs_per_call) < 1:
            raise ValueError("pairs_per_call must be >= 1, got %r" % (pairs_per_call,))
        self.shutter_angle, self.shutter_samples = _shutter_angle(shutter_angle), _shutter_samples(shutter_samples)
        super().__init__(model, ds_factor, bgr, pairs_per_call, scene_threshold)
        self.fps_in, self.fps_out = _rate(fps_in, "fps_in"), _rate(fps_out, "fps_out")
        self.step = self.fps_in / self.fps_out   # input frames per output frame
        # the exposure window in input frames (None: no shutter)
        self.window = None if self.shutter_angle is None else self.shutter_angle / 360 * self.step

    def reset(self):
        super().reset()
        self._k = 0             # next output index to schedule

    @staticmethod
    def _instant(j: int, x: Fraction):
        """an instant x in (j - 1, j] -> (its offset in (0, 1], the float32 t of its query or None for an input frame)"""
        off = x - (j - 1)
        # input frame j, or (a hair after it) frame j - 1; any other instant is interpolated at the float32 t the engine receives
        return off, None if off >= 1 - SNAP or off <= SNAP else float(np.float32(float(off)))

    def _instants(self, j: int):
        while self._k * self.step <= j:   # the output instants in (j - 1, j] (frame 0: the instant 0)
            x = self._k * self.step
            self._k += 1
            yield self._instant(j, x)

    def _schedule(self, j: int, prev_u8, frame_u8, cur_u8):
        if self.window is None:
            return super()._schedule(j, prev_u8, frame_u8, cur_u8)
        w, S = self.window, self.shutter_samples
        # every output whose window starts by frame j, so that each sample in (j - 1, j] is placed now
        while self._k * self.step - w / 2 + w / (2 * S) <= j:
            tau = self._k * self.step
            inst = [tau - w / 2 + (2 * i + 1) * w / (2 * S) for i in range(S)]
            self._queue.append(_Entry(pending=inst, needs=math.ceil(inst[-1]) if S > 1 else 0, tau=tau))
            self._k += 1
        for e in self._queue:
            while e.pending and e.pending[0] <= j:
                x = e.pending.pop(0)
                if x < 0:   # before frame 0
                    continue
                s = self._sample(j, *self._instant(j, x), prev_u8, frame_u8, cur_u8)
                e.samples.append(s)
                if x == e.tau:
                    e.own = s

    def _end_clip(self):
        if self.window is None:
            return
        last = self._n - 1
        self._queue = [e for e in self._queue if e.tau <= last]
        for e in self._queue:
            e.pending = []    # the samples after the last frame
        self._ended = True

    def _preds(self, ims: torch.Tensor):
        if self.window is None:
            return super()._preds(ims)
        return ims.contiguous().unbind(0)   # the sub-frames stay padded float until their outputs are blended

    def _kept(self, e: _Entry) -> List[_Sample]:
        """the samples of a complete entry in its own shot: no cut between a sample's frame (a pair: its first frame) and the own one's"""
        if self._scene is None or len(e.samples) == 1:
            return e.samples
        pos = lambda s: s.f if s.pair is None else s.pair[0]
        own = pos(e.own)
        return [s for s in e.samples if not any(c in self._scene for c in range(min(pos(s), own) + 1, max(pos(s), own) + 1))]

    def _output(self, e: _Entry) -> torch.Tensor:
        if self.window is None:
            return super()._output(e)
        return blend_u8([s.out if s.pair is not None else s.u8 for s in self._kept(e)], self._padder, self.bgr)

    def _run(self, used, frames, queries):
        return self.model._interpolate_at(torch.stack(frames, 0), queries, self.ds, False)["imgt_pred"], None
