"""Drop-in ``GIMMVFI_F`` boundary (reference: src/models/generalizable_INR/gimmvfi_f.py:27-484): same constructor argument, the 639-key
``state_dict`` of the reference (FlowFormer included, so published GIMM-VFI-F / F-P checkpoints load with ``strict=True``), same
``forward(img_xs, coord, t, ds_factor)`` and returned dict.

Everything runs natively on the sm_90a engine (``gimmvfi_finalize_weights_f`` + ``gimmvfi_forward``):
  * the FlowFormer flow estimator (gimmvfi_f.py:114-138 -> LatentCostFormer/transformer.py:45-74): Twins-SVT-L encoders, cost-perceiver
    memory encoder, 32-iteration GMA memory decoder — csrc/flowformer.cu + csrc/ops_tokens.cu, both directions batched;
  * everything downstream of ``cal_bidirection_flow`` — the same kernels as GIMM-VFI-R (F has no feature projections,
    gimmvfi_f.py:37-60).
``model.flow_backend`` (optional) swaps the estimator for a caller-supplied callable with the signature of the reference's
``FlowFormer.forward(im0, im1, return_feat=True)``; ``forward(..., flow_inputs=...)`` takes precomputed estimator outputs
(``gimmvfi_forward_from_flow``).  There is no PyTorch re-implementation of FlowFormer on the product path."""
from typing import Callable, Optional

import torch

from .arch import ESTIMATOR_PREFIX, param_spec_f
from .model import _VFIBase
from .weights import random_state_dict_f


class GIMMVFI_F(_VFIBase):
    def __init__(self, config=None, seed: int = 0):
        super().__init__(config, full_f=True)
        self.raft_iter = getattr(self.config, "raft_iter", 20)
        self.build_params(param_spec_f(), random_state_dict_f(seed))
        self.flow_backend: Optional[Callable] = None   # see the module docstring

    def flow_estimator_state_dict(self) -> dict:
        """`flow_estimator.*` with the prefix stripped: what the reference FlowFormer module's load_state_dict takes."""
        return {k[len(ESTIMATOR_PREFIX):]: v for k, v in self.state_dict().items() if k.startswith(ESTIMATOR_PREFIX)}

    def cal_bidirection_flow(self, im0, im1):
        """gimmvfi_f.py:114-138 through an EXTERNAL flow backend (model.flow_backend) -> the dict gimmvfi_forward_from_flow takes.
        Without a backend forward() runs the engine's native FlowFormer and never calls this."""
        assert self.flow_backend is not None
        f01, feats0, fnet0 = self.flow_backend(im0, im1)
        f10, feats1, fnet1 = self.flow_backend(im1, im0)
        f01 = f01[0] if isinstance(f01, (list, tuple)) else f01
        f10 = f10[0] if isinstance(f10, (list, tuple)) else f10
        return dict(flows=torch.stack([f01, f10], 2), feat4=[feats0[0], feats1[0]], feat8=[feats0[1], feats1[1]], fnet=[fnet0, fnet1])

    def _external_flows(self, xs, ds_factor):
        if self.flow_backend is None:
            return None
        x_net = xs
        if ds_factor is not None:   # gimmvfi_f.py:309-318: the estimator sees the down-scaled frames
            rs = lambda a: torch.nn.functional.interpolate(a, scale_factor=ds_factor, mode="bilinear", align_corners=False)
            x_net = torch.stack([rs(xs[:, :, 0]), rs(xs[:, :, 1])], 2)
        return self.cal_bidirection_flow(255 * x_net[:, :, 0], 255 * x_net[:, :, 1])

    @torch.no_grad()
    def forward(self, img_xs, coord=None, t=None, ds_factor=None, flow_inputs=None):
        """gimmvfi_f.py:304-384 (inference form).  `flow_inputs` (optional) = precomputed outputs of cal_bidirection_flow."""
        self._check_args(coord, t)
        return self._interpolate(img_xs, coord, t, ds_factor, self.aux_outputs, flow_inputs=flow_inputs)
