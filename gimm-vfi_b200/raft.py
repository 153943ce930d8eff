"""Drop-in ``RAFT`` for inference (reference: raft/raft.py:26-169, the optical-flow estimator GIMM-VFI-R builds with initialize_RAFT(),
raft/__init__.py:7-24) — the estimator alone, on any frame pairs.  Same ``state_dict`` as the reference module (GIMM-VFI-R's
``flow_estimator.*`` with the prefix stripped, ``norm3`` and ``downsample.1`` one module as in raft/extractor.py:44-47; loads with
``strict=True``), same ``forward(image1, image2, iters=12, flow_init=None, upsample=True, test_mode=False, return_feat=True)`` with the
reference's three return forms; ``flows(frames, pairs)`` runs a whole pair list over a frame set as ONE engine call, where fnet encodes
every frame once and cnet every source frame once however many pairs use it.  Everything runs in the sm_90a engine (csrc/engine.cu
run_raft, the estimator of GIMM-VFI-R), in the engine's arithmetic: ``args.mixed_precision`` and ``args.alternate_corr`` are accepted
and change nothing (the correlation is the volume pyramid, or the volume-free lookup when a pair list's pyramid would not fit the
device).  CUDA only.

Memory per pair: the volume pyramid is N^2 * 4/3 floats, N = (H/8)(W/8): 0.5 GB at 544x960, 8.5 GB at 1088x1920."""
from typing import Sequence, Tuple

import torch

from .arch import ESTIMATOR_PREFIX, param_spec_r, strip_prefix
from .engine import EngineHandle
from .module import EngineModule, load_estimator_checkpoint
from .weights import random_state_dict

load_raft_checkpoint = load_estimator_checkpoint


def param_spec_raft():
    """(key, shape, dtype) of the reference RAFT module: GIMM-VFI-R's flow_estimator.* in registration order, prefix stripped"""
    return strip_prefix(param_spec_r())


def raft_forward(eng: EngineHandle, image1, image2, iters=12, flow_init=None, test_mode=False, return_feat=True):
    """RAFT.forward (raft.py:100-169) through an engine that serves RAFT: image1, image2 (B,3,H,W) in [0,255], H and W multiples of 8 and
    >= 128; the B rows are B pairs in one engine call.  test_mode -> (flow_low, flow_up); else return_feat -> (flow_up, [feat4, feat8],
    fmap1); else the list of `iters` upsampled flows (flow_predictions)."""
    if image1.shape != image2.shape or image1.dim() != 4 or image1.shape[1] != 3:
        raise ValueError("RAFT: image1 and image2 must both be (B,3,H,W), got %s and %s" % (tuple(image1.shape), tuple(image2.shape)))
    B = image1.shape[0]
    frames = torch.cat([image1, image2], 0).to(torch.float32).contiguous()
    pairs = [(b, B + b) for b in range(B)]
    if test_mode:
        o = eng.raft_forward(frames, pairs, iters, flow_init, outputs=("flow_up", "flow_low"))
        return o["flow_low"], o["flow_up"]
    if return_feat:
        o = eng.raft_forward(frames, pairs, iters, flow_init, outputs=("flow_up", "feat4", "feat8", "fmap"))
        return o["flow_up"], [o["feat4"], o["feat8"]], o["fmap"]
    o = eng.raft_forward(frames, pairs, iters, flow_init, outputs=("flow_iters",))
    return list(o["flow_iters"].unbind(0))


class RAFT(EngineModule):
    def __init__(self, args=None, seed: int = 0):
        super().__init__(raft=True)
        if args is not None and getattr(args, "small", False):
            raise NotImplementedError("RAFT (gimmvfi_b200): args.small=True is RAFT-small, a different network; the engine builds the full "
                                      "RAFT of GIMM-VFI-R (raft.py:38-44, 64-70)")
        self.args = args
        self.hidden_dim = self.context_dim = 128
        self.build_params(param_spec_raft(), random_state_dict(seed), ESTIMATOR_PREFIX)
        # 4 (default, as GIMM-VFI-R): RAFT on the fp32-class 3xF16 / 3xTF32 tensor-core forms; 0: fp32 CUDA cores
        self.tensor_cores = 4

    @torch.no_grad()
    def forward(self, image1, image2, iters=12, flow_init=None, upsample=True, test_mode=False, return_feat=True):
        """raft.py:100-169.  image1, image2 (B,3,H,W) in [0,255] -> test_mode: (flow_low (B,2,H/8,W/8), flow_up (B,2,H,W)); return_feat:
        (flow_up, [feat4 (B,96,H/4,W/4), feat8 (B,128,H/8,W/8)], fmap1 (B,256,H/8,W/8)); neither: a list of `iters` (B,2,H,W) flows.
        flow_init (B,2,H/8,W/8) warm-starts coords1.  `upsample` is ignored, as in the reference."""
        return raft_forward(self._ready(image1), image1, image2, iters, flow_init, test_mode, return_feat)

    @torch.no_grad()
    def flows(self, frames: torch.Tensor, pairs: Sequence[Tuple[int, int]], iters: int = 12, flow_init=None, flow_low: bool = False):
        """Pair-list form: frames (F,3,H,W) in [0,255], pairs [(source, target), ...] -> flow_up (P,2,H,W) from each source to its target
        [, flow_low (P,2,H/8,W/8)].  Pair (s, t) equals forward(frames[s:s+1], frames[t:t+1], iters, flow_init[p:p+1], test_mode=True)."""
        if len(pairs) == 0:
            raise ValueError("RAFT.flows: at least one pair is required")
        frames = frames.to(torch.float32).contiguous()
        o = self._ready(frames).raft_forward(frames, pairs, iters, flow_init, outputs=("flow_up", "flow_low") if flow_low else ("flow_up",))
        return (o["flow_up"], o["flow_low"]) if flow_low else o["flow_up"]
