"""Drop-in ``GIMM`` for inference (reference: src/models/generalizable_INR/gimm.py:25-253) — the motion-modelling network
alone: bidirectional flows in, the normalised flow at time t out (SURVEY.md 8(f) row 4).  Same constructor argument, same
``forward(xs, coord, keep_xs_shape, ori_flow, timesteps)`` signature, same 36-key ``state_dict``; ``forward`` is one call
into the sm_90a engine (the kernels of the GIMM stages of GIMM-VFI-R, csrc/engine.cu gimm_encode / gimm_decode).  CUDA only."""
import torch

from .arch import param_spec_r
from .engine import EngineHandle
from .model import _GIMMBase
from .weights import random_state_dict

GIMM_KEY_PREFIXES = ("g_filter", "alpha_v", "alpha_fe", "cnn_encoder.", "res_conv.", "hyponet.")


def param_spec_gimm():
    """(key, shape, dtype) of gimm.py's module tree in the reference's registration order (gimm.py:36-80):
    g_filter, alpha_v, alpha_fe, cnn_encoder.*, res_conv.*, hyponet.*  — the same names GIMM-VFI-R uses (gimmvfi_r.py:86-111)."""
    spec = [e for e in param_spec_r() if e[0].startswith(GIMM_KEY_PREFIXES)]
    order = {p: i for i, p in enumerate(GIMM_KEY_PREFIXES)}
    rank = lambda k: next(order[p] for p in GIMM_KEY_PREFIXES if k.startswith(p))
    return sorted(spec, key=lambda e: rank(e[0]))   # stable: keeps the order inside each group


class GIMM(_GIMMBase):
    def __init__(self, config=None, seed: int = 0):
        super().__init__(config, gimm_only=True)
        self.build_params(param_spec_gimm(), random_state_dict(seed))
        self.tensor_cores = 1   # 0: fp32 CUDA cores; >= 1: TF32 wgmma (everything here is downstream of RAFT, DESIGN.md precision plan)

    @torch.no_grad()
    def forward(self, xs, coord=None, keep_xs_shape=True, ori_flow=None, timesteps=None):
        """gimm.py:129-214.  xs (B,2,2,H,W) normalised flows, ori_flow (B,2,2,H,W) raw flows, coord (B,1,Hc,Wc,3) on a grid of
        any size (e.g. sample_coord_input(..., upsample_ratio=r): Hc = int(H r)); list form (timesteps and coord lists of equal
        length) -> list of outputs, tensor form -> one output; (B,2,1,Hc,Wc) with keep_xs_shape else (B,1,Hc,Wc,2).
        In the list form the grids may differ in size: one engine call per distinct size (see gimm_forward_grids)."""
        if coord is None or ori_flow is None or timesteps is None:
            raise ValueError("GIMM.forward needs coord, ori_flow and timesteps (the reference's coord=None default cannot run either, gimm.py:132)")
        eng = self._ready(xs)
        is_list = isinstance(timesteps, list)
        if is_list:
            assert isinstance(coord, list)
            assert len(timesteps) == len(coord)
        cl, tl = (coord, timesteps) if is_list else ([coord], [timesteps])
        out = gimm_forward_grids(eng, xs, ori_flow, cl, tl)   # [(B,2,1,Hc,Wc)]
        outs = [o if keep_xs_shape else o.permute(0, 2, 3, 4, 1) for o in out]
        return outs if is_list else outs[0]


def gimm_forward_grids(eng: EngineHandle, xs, ori_flow, coords, timesteps):
    """GIMM.forward's list form on an engine: coords [(B,1,Hc,Wc,3)], timesteps [(B,) or scalar] -> [(B,2,1,Hc,Wc)] in the same order.
    Every grid may have its own size (the reference resizes the latent per grid, hyponet.py:86-90).  Timesteps that share a grid size
    go into one engine call; each further distinct size is one more call, which recomputes the t-independent encoder: correct, not
    optimised for mixed sizes."""
    B = xs.shape[0]
    xs = xs.to(torch.float32).contiguous()
    ori_flow = ori_flow.to(torch.float32).contiguous()
    groups = {}   # grid size -> indices, in the order the sizes first appear
    for i, c in enumerate(coords):
        groups.setdefault(tuple(c.shape[-3:-1]), []).append(i)
    outs = [None] * len(coords)
    for idx in groups.values():
        cs = torch.stack([coords[i].to(torch.float32) for i in idx], 0).contiguous()
        tt = torch.stack([timesteps[i].reshape(-1).to(torch.float32).expand(B) for i in idx], 0).contiguous()
        out = eng.gimm_forward(xs, ori_flow, cs, tt)   # (T,B,2,1,Hc,Wc)
        for j, i in enumerate(idx):
            outs[i] = out[j]
    return outs
