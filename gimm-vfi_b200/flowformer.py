"""Drop-in ``FlowFormer`` for inference (reference: flowformer/core/FlowFormer/LatentCostFormer/transformer.py:29-74, the optical-flow
estimator GIMM-VFI-F builds with initialize_Flowformer(), flowformer/__init__.py) — the estimator alone, on any frame pairs.  Same
``state_dict`` as the reference module (GIMM-VFI-F's ``flow_estimator.*`` with the prefix stripped; loads with ``strict=True``), same
``forward(image1, image2)`` returning ``(flow_up, flow_low)``; ``flows(frames, pairs)`` runs a whole pair list over a frame set as ONE
engine call, where every frame is encoded once however many pairs use it.  Everything runs in the sm_90a engine (csrc/flowformer.cu,
the estimator of GIMM-VFI-F).  CUDA only.

Memory per pair: the cost volume and the GMA attention matrix are N^2 floats each, N = (H/8)(W/8): 12.8 MB each at 256x448,
4.3 GB each at 1088x1920.  A caller bounds the number of pairs per call accordingly."""
from typing import Optional, Sequence, Tuple

import torch

from .arch import ESTIMATOR_PREFIX, param_spec_f, strip_prefix
from .module import EngineModule, load_estimator_checkpoint
from .weights import random_state_dict_f

load_flowformer_checkpoint = load_estimator_checkpoint


def param_spec_flowformer():
    """(key, shape, dtype) of the reference FlowFormer module: GIMM-VFI-F's flow_estimator.* in registration order, prefix stripped"""
    return strip_prefix(param_spec_f())


class FlowFormer(EngineModule):
    def __init__(self, cfg=None, seed: int = 0):
        super().__init__(flowformer=True)
        self.cfg = cfg
        self.build_params(param_spec_flowformer(), random_state_dict_f(seed), ESTIMATOR_PREFIX)
        # 4 (default): the 3xF16 fp32-class tensor-core forms, ~2e-3 px from the reference; 0: fp32 CUDA cores, ~2e-4 px
        self.tensor_cores = 4

    @torch.no_grad()
    def forward(self, image1, image2, output=None, flow_init=None, return_feat=False, iters=None) -> Tuple[torch.Tensor, torch.Tensor]:
        """transformer.py:45-74: image1, image2 (B,3,H,W) in [0,255], H and W multiples of 32 -> (flow_up (B,2,H,W), flow_low
        (B,2,H/8,W/8)).  The B pairs form one reference call, including the batch order in which the reference hands the context to
        the cost memory (twins.py:367, context.repeat)."""
        if output is not None or flow_init is not None or return_feat:
            raise NotImplementedError("FlowFormer (gimmvfi_b200): output, flow_init and return_feat=True are not on the inference path")
        if image1.shape != image2.shape or image1.dim() != 4:
            raise ValueError("FlowFormer: image1 and image2 must both be (B,3,H,W), got %s and %s" % (tuple(image1.shape), tuple(image2.shape)))
        B = image1.shape[0]
        frames = torch.cat([image1, image2], 0).to(torch.float32).contiguous()
        eng = self._ready(frames)
        return eng.flowformer_forward(frames, [(b, B + b) for b in range(B)], pairs_per_call=B, iters=int(iters or 0), flow_low=True)

    @torch.no_grad()
    def flows(self, frames: torch.Tensor, pairs: Sequence[Tuple[int, int]], iters: Optional[int] = None, flow_low: bool = False):
        """Pair-list form: frames (F,3,H,W) in [0,255], pairs [(source, target), ...] -> flow_up (P,2,H,W) from each source to its
        target [, flow_low (P,2,H/8,W/8)].  Every pair equals FlowFormer.forward(frames[source:source+1], frames[target:target+1])."""
        if len(pairs) == 0:
            raise ValueError("FlowFormer.flows: at least one pair is required")
        frames = frames.to(torch.float32).contiguous()
        eng = self._ready(frames)
        return eng.flowformer_forward(frames, pairs, pairs_per_call=1, iters=int(iters or 0), flow_low=flow_low)
