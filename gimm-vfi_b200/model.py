"""Drop-in ``GIMMVFI_R`` for inference (reference: src/models/generalizable_INR/
gimmvfi_r.py:34-507).  Same constructor argument (``config.arch`` node), same
``forward(img_xs, coord, t, iters, ds_factor)`` signature and returned dict, same
414-key ``state_dict`` — but ``forward`` is one call into the sm_90a engine through
the C ABI.  CUDA only; there is no PyTorch / CPU fallback path.
"""
import numpy as np
import torch
import torch.nn as nn

from .arch import param_spec_r
from .config import default_arch_config
from .engine import AUX_OUTPUTS, EngineHandle, aux_keys, model_outputs
from .module import EngineModule, _RootRef
from .weights import random_state_dict


class _FlowEstimator(nn.Module):
    """GIMMVFI_R.flow_estimator: the RAFT module's parameter tree (gimmvfi_r.py:45), callable with RAFT.forward (raft/raft.py:100-169)
    through the model's own engine, so the weights are not loaded twice.  The model is held by a _RootRef, not registered as a
    submodule: the state_dict, its order and its sharing are the reference's."""

    hidden_dim = context_dim = 128

    def __init__(self, model):
        super().__init__()
        self.__dict__["_model"] = _RootRef(model)

    @torch.no_grad()
    def forward(self, image1, image2, iters=12, flow_init=None, upsample=True, test_mode=False, return_feat=True):
        """RAFT.forward's three return forms, as gimmvfi_b200.RAFT.forward; `upsample` is ignored, as in the reference."""
        from .raft import raft_forward

        return raft_forward(self.__dict__["_model"]()._ready(image1), image1, image2, iters, flow_init, test_mode, return_feat)


def sample_coords(batch_size, s_shape, t_ids, coord_range=(-1.0, 1.0), upsample_ratio=1.0, device=None):
    """CoordSampler3D.shape2coordinate (modules/coord_sampler.py:21-43): (B, T, Hc, Wc, 3), last dim (t, y, x)."""
    assert isinstance(t_ids, list)
    cs = [(torch.tensor(t_ids, device=device) / 1.0).to(torch.float32)]
    for n in s_shape:
        n = int(n * upsample_ratio)
        c = (0.5 + torch.arange(n, device=device)) / n
        cs.append(coord_range[0] + (coord_range[1] - coord_range[0]) * c)
    g = torch.stack(torch.meshgrid(*cs, indexing="ij"), dim=-1)
    return g.unsqueeze(0).repeat(batch_size, 1, 1, 1, 1)


class _GIMMBase(EngineModule):
    """GIMM, GIMMVFI_R and GIMMVFI_F: the `config.arch` node they are built from and the reference's sample_coord_input."""

    def __init__(self, config, **weight_set):
        super().__init__(**weight_set)
        self.config = config = (config.copy() if config is not None else default_arch_config())
        self.hyponet_config = config.hyponet
        self.fwarp_type = getattr(config, "fwarp_type", "linear")
        self._motion = motion_settings(config)
        self.coord_range = list(config.coord_range)

    def _motion_config(self):
        return self._motion

    def sample_coord_input(self, batch_size, s_shape, t_ids, coord_range=None, upsample_ratio=1.0, device=None):
        """gimm.py:239-253, gimmvfi_r.py:428-442, gimmvfi_f.py:391-407"""
        assert device is not None
        assert coord_range is None
        return sample_coords(batch_size, s_shape, t_ids, self.coord_range, upsample_ratio, device)


class _VFIBase(_GIMMBase):
    """GIMMVFI_R and GIMMVFI_F: a whole interpolation is one engine forward, returning the reference's dict."""

    # whether the engine runs RAFT's encoders, whose products a frame cache keeps (GIMMVFI_R).  Without them the cache would do nothing
    # but turn off the engine's CUDA-graph replay, so _interpolate does not hand it on.
    _raft_encoders = False

    def __init__(self, config, **weight_set):
        super().__init__(config, **weight_set)
        self.num_flows = 3
        # True: every auxiliary output; False: imgt_pred only; or a collection of keys of the returned dict, e.g. ("flowt",):
        # imgt_pred plus those (the engine allocates and writes only what is selected)
        self.aux_outputs = True
        # 0: fp32 CUDA cores everywhere; 1: post-RAFT convolutions on wgmma TF32 (RAFT on CUDA cores);
        # 2: additionally RAFT + correlation on wgmma with 3xTF32 operand splitting and register-promoted accumulation
        # (fp32-class accuracy); 3: additionally the final decoder's 256-channel residual trunk stored in fp16 and run on f16
        # MMAs (same 10-bit mantissa as TF32); 4 (default): additionally the 32/64-channel full-resolution chains, the init-decoder
        # trunk and the decoder concat in fp16 storage.  All modes meet max|d imgt_pred| <= 1e-3 vs the reference.
        self.tensor_cores = 4

    @staticmethod
    def _check_args(coord, t):
        """the inference form of the reference forward's coord and t (gimmvfi_r.py:324-367, gimmvfi_f.py:304-343)"""
        assert isinstance(t, list)
        assert isinstance(coord, list)
        assert len(t) == len(coord)
        for c in coord:
            assert isinstance(c, tuple)
            if c[1] is not None:
                raise NotImplementedError("sub-sampled coordinates are the training path (gimmvfi_r.py:358-367, gimmvfi_f.py:334-343); "
                                          "inference passes None")

    def _external_flows(self, xs, ds_factor):
        """flow_inputs for the engine when the estimator runs outside it (GIMMVFI_F.flow_backend); None: the engine's own"""
        return None

    def _interpolate(self, img_xs, coord, t, ds_factor, aux, frame_cache=None, flow_inputs=None):
        """forward's body.  aux: an aux_outputs selection; frame_cache: see EngineHandle.forward, used by GIMMVFI_R only (the RAFT
        encoders' products); flow_inputs: precomputed estimator outputs, as GIMMVFI_F.cal_bidirection_flow returns them."""
        eng = self._ready(img_xs)
        B = img_xs.shape[0]
        xs = img_xs.to(torch.float32).contiguous()
        if flow_inputs is None:
            flow_inputs = self._external_flows(xs, ds_factor)
        coords = torch.stack([c[0].to(torch.float32) for c in coord], 0).contiguous()  # (T,B,1,Hc,Wc,3)
        tt = torch.stack([x.reshape(-1).to(torch.float32).expand(B) for x in t], 0).contiguous()  # (T,B)
        keys = aux_keys(aux)
        o = eng.forward(xs, coords, tt, ds_factor, aux_outputs=[f for k in keys for f in AUX_OUTPUTS[k]],
                        frame_cache=frame_cache if self._raft_encoders else None, flow_inputs=flow_inputs)
        return model_outputs(o, len(t), keys)

    @staticmethod
    def _check_clip_args(frames, pairs, t):
        """interpolate's arguments -> (pairs as int tuples, t as floats); raises ValueError before any engine work"""
        if not torch.is_tensor(frames) or frames.dim() != 4 or frames.shape[1] != 3 or frames.shape[0] < 1:
            raise ValueError("interpolate: frames must be a (F,3,H,W) tensor with F >= 1, got %s"
                             % (tuple(frames.shape) if torch.is_tensor(frames) else type(frames).__name__,))
        F = frames.shape[0]
        try:
            pl = [(int(a), int(b)) for a, b in pairs]
        except (TypeError, ValueError):
            raise ValueError("interpolate: pairs must be a sequence of (source, target) frame indices")
        if not pl:
            raise ValueError("interpolate: the pair list is empty")
        bad = [ab for ab in pl if not (0 <= ab[0] < F and 0 <= ab[1] < F)]
        if bad:
            raise ValueError("interpolate: pair(s) %s index outside the %d frames" % (bad, F))
        if not isinstance(t, (list, tuple)) or not t:
            raise ValueError("interpolate: t must be a non-empty list of floats (the timesteps every pair is interpolated at)")
        try:
            ts = [float(x) for x in t]
        except (TypeError, ValueError):
            raise ValueError("interpolate: t must be a list of floats, one per timestep")
        return pl, ts

    @torch.no_grad()
    def interpolate(self, frames, pairs, t, ds_factor=None):
        """A clip in one engine call: frames (F,3,H,W) in [0,1], pairs [(src, tgt), ...] of frame indices (any: reversed, repeated, a
        frame with itself), t a list of T floats shared by every pair.  Returns forward()'s dict with the pair axis in place of the batch
        axis, under the same aux_outputs selection: pair p is forward() on (frames[src], frames[tgt]).  Each frame is resized and encoded
        once however many pairs use it; the coordinates are sample_coord_input's at the network resolution."""
        return self._interpolate_clip(frames, pairs, t, ds_factor, self.aux_outputs)

    def _interpolate_clip(self, frames, pairs, t, ds_factor, aux):
        """interpolate's body; aux: an aux_outputs selection"""
        pl, ts = self._check_clip_args(frames, pairs, t)
        if getattr(self, "flow_backend", None) is not None:
            raise NotImplementedError("interpolate runs the engine's own flow estimator; model.flow_backend is only used by forward()")
        eng = self._ready(frames)
        x = frames.to(torch.float32).contiguous()
        P, (Hf, Wf) = len(pl), x.shape[-2:]
        ratio = 1.0 if ds_factor is None else ds_factor
        coords = torch.stack([self.sample_coord_input(P, (Hf, Wf), [ti], device=x.device, upsample_ratio=ratio) for ti in ts], 0)
        tt = torch.tensor(ts, dtype=torch.float32, device=x.device).unsqueeze(1).expand(len(ts), P).contiguous()
        keys = aux_keys(aux)
        o = eng.forward_clip(x, pl, coords.to(torch.float32).contiguous(), tt, ds_factor,
                             aux_outputs=[f for k in keys for f in AUX_OUTPUTS[k]])
        return model_outputs(o, len(ts), keys)

    @staticmethod
    def _check_query_args(frames, queries):
        """interpolate_at's arguments -> [(src, tgt, t)] as (int, int, float); raises ValueError before any engine work"""
        if not torch.is_tensor(frames) or frames.dim() != 4 or frames.shape[1] != 3 or frames.shape[0] < 1:
            raise ValueError("interpolate_at: frames must be a (F,3,H,W) tensor with F >= 1, got %s"
                             % (tuple(frames.shape) if torch.is_tensor(frames) else type(frames).__name__,))
        F = frames.shape[0]
        try:
            ql = [(int(a), int(b), float(t)) for a, b, t in queries]
        except (TypeError, ValueError):
            raise ValueError("interpolate_at: queries must be a sequence of (source, target, t)")
        if not ql:
            raise ValueError("interpolate_at: the query list is empty")
        bad = [q for q in ql if not (0 <= q[0] < F and 0 <= q[1] < F)]
        if bad:
            raise ValueError("interpolate_at: query(s) %s index outside the %d frames" % (bad, F))
        # strictly inside (0, 1) as the float32 the engine receives: the AMT correlation lookup divides by t and 1 - t
        # (gimmvfi_r.py:494-507); NaN fails both comparisons
        with np.errstate(over="ignore"):
            bad = [q for q in ql if not (0.0 < float(np.float32(q[2])) < 1.0)]
        if bad:
            raise ValueError("interpolate_at: query(s) %s have t outside the open interval (0, 1) in float32" % (bad,))
        return ql

    @torch.no_grad()
    def interpolate_at(self, frames, queries, ds_factor=None):
        """Every pair at its own timesteps, in one engine call: frames (F,3,H,W) in [0,1], queries [(src, tgt, t), ...] with t strictly
        inside (0, 1).  The queries of one (src, tgt) are that pair's timesteps, in query order; each used frame is encoded once, and each
        distinct pair's estimator runs once.  Query q's result is forward() with B = 1 on (frames[src], frames[tgt]) at its pair's own
        timestep list, the coordinates sample_coord_input's at the network resolution.  Returns a dict keyed by engine output name:
        imgt_pred (Q,3,H,W) and the outputs the aux_outputs selection maps to (AUX_OUTPUTS), per-timestep ones with the query axis first,
        raft_flow / nflow (P,2,2,h,w) over the distinct pairs; plus pairs (the P distinct (src, tgt) in first-appearance order) and
        pair_index (Q,), each query's index among them."""
        return self._interpolate_at(frames, queries, ds_factor, self.aux_outputs)

    def _interpolate_at(self, frames, queries, ds_factor, aux):
        """interpolate_at's body; aux: an aux_outputs selection"""
        ql = self._check_query_args(frames, queries)
        if getattr(self, "flow_backend", None) is not None:
            raise NotImplementedError("interpolate_at runs the engine's own flow estimator; model.flow_backend is only used by forward()")
        eng = self._ready(frames)
        x = frames.to(torch.float32).contiguous()
        keys = aux_keys(aux)
        out = eng.forward_queries(x, ql, ds_factor, aux_outputs=[f for k in keys for f in AUX_OUTPUTS[k]], coord_range=self.coord_range)
        pairs, index = eng.query_pairs(ql)
        out["pairs"] = pairs
        out["pair_index"] = torch.tensor(index, dtype=torch.int64)
        return out

    def compute_psnr(self, preds, targets, reduction="mean"):
        """gimmvfi_r.py:412-426 (the same in gimmvfi_f.py)"""
        assert reduction in ["mean", "sum", "none"]
        mse = torch.reshape((preds - targets) ** 2, (preds.shape[0], -1)).mean(dim=-1)
        psnr = -10 * torch.log10(mse)
        return psnr.mean() if reduction == "mean" else (psnr.sum() if reduction == "sum" else psnr)


class GIMMVFI_R(_VFIBase):
    _raft_encoders = True

    def __init__(self, config=None, seed: int = 0):
        super().__init__(config)
        self.raft_iter = 20  # gimmvfi_r.py:41 (config.raft_iter is ignored by the reference too)
        self.flow_estimator = _FlowEstimator(self)   # the first child in the reference's order; build_params fills it
        self.build_params(param_spec_r(), random_state_dict(seed))

    @torch.no_grad()
    def forward(self, img_xs, coord=None, t=None, iters=None, ds_factor=None):
        """gimmvfi_r.py:324-407 (inference form).  ``iters`` is accepted and ignored, as in
        the reference (cal_bidirection_flow hard-codes 20, gimmvfi_r.py:126-132)."""
        self._check_args(coord, t)
        return self._interpolate(img_xs, coord, t, ds_factor, self.aux_outputs)

    def warp_frame(self, frame, flow):
        """gimmvfi_r.py:409-410 — backward warp of an NCHW frame by an NCHW flow."""
        import ctypes as C

        from ._lib import default_lib, view_of

        lib = default_lib()
        src = frame.to(torch.float32).permute(0, 2, 3, 1).contiguous()
        fl = flow.to(torch.float32).permute(0, 2, 3, 1).contiguous()
        dst = torch.empty(fl.shape[0], fl.shape[1], fl.shape[2], src.shape[3], device=src.device)
        s = C.c_void_p(torch.cuda.current_stream(src.device).cuda_stream)
        lib.check(lib.dll.gimmvfi_op_backwarp(C.byref(view_of(src)), C.byref(view_of(fl)), C.byref(view_of(dst)), s))
        return dst.permute(0, 3, 1, 2).contiguous()


def motion_settings(config) -> dict:
    """EngineHandle.set_motion_config's arguments from an `arch` config: fwarp_type (gimm.py:144-157, softsplat.py:286-352 with
    "-zeroeps" appended) and HypoNet's activation (modules/utils.py:65-76), siren_w0, output_bias and normalize_weight (hyponet.py:
    127-143).  Missing keys take the shipped values.  fwarp_type "avg" is refused: the reference normalises by the last latent channel
    there, and res_conv then fails on the channel count."""
    fwarp = getattr(config, "fwarp_type", "linear")
    if fwarp == "avg":
        raise NotImplementedError("fwarp_type='avg': the reference cannot run it (softsplat 'avg-zeroeps' appends no ones channel, so the "
                                  "splat loses a latent channel and res_conv refuses the 30 + 32 channel input)")
    if fwarp not in EngineHandle.FWARP_MODES:
        raise NotImplementedError("fwarp_type=%r: softsplat knows linear, softmax, sum and avg" % (fwarp,))
    hy = config.hyponet
    act = getattr(hy, "activation", None)
    kind = getattr(act, "type", "siren") if act is not None else "siren"
    if kind not in EngineHandle.ACTIVATIONS:
        raise NotImplementedError("hyponet.activation.type=%r: create_activation knows relu, siren, silu and damp" % (kind,))
    w0 = getattr(act, "siren_w0", 1.0) if act is not None else 1.0
    if kind in ("siren", "damp") and w0 is None:
        raise ValueError("hyponet.activation.siren_w0 is required by %s" % kind)
    return dict(fwarp_type=fwarp, activation=kind, w0=float(w0) if w0 is not None else 1.0,
                output_bias=float(getattr(hy, "output_bias", 0.5)), normalize_weight=bool(getattr(hy, "normalize_weight", True)))


def _check_engine_config(config):
    """The engine is specialised to HypoNet's shipped shape (configs/gimmvfi/*.yaml, module_config.py:28-41): a config that asks for
    another parameter shape or kernel tile must fail here, not be silently ignored.  The settings that change no shape (fwarp_type,
    activation, siren_w0, output_bias, normalize_weight) are honoured: motion_settings."""
    hy = config.hyponet
    want = dict(type="mlp", n_layer=5, input_dim=3, output_dim=2, use_bias=True)
    for k, v in want.items():
        if getattr(hy, k, v) != v:
            raise NotImplementedError("hyponet.%s=%r: the sm_90a engine is built for the shipped value %r" % (k, getattr(hy, k), v))
    if list(getattr(hy, "hidden_dim", [128])) != [128]:
        raise NotImplementedError("hyponet.hidden_dim=%r: the engine is built for [128]" % (list(hy.hidden_dim),))
    motion_settings(config)
    if getattr(config, "modulated_layer_idxs", None) not in (None, [], [1]):
        raise NotImplementedError("modulated_layer_idxs: weight modulation is unused by the shipped models (hyponet.py:101-117 is a no-op)")


def create_model(config, ema: bool = False):
    """src/models/__init__.py:15-37 for the three model types (gimmvfi_r, gimmvfi_f, gimm)."""
    model_type = config.type.lower()
    if ema:
        raise NotImplementedError("EMA wrappers are training-only (src/models/ema.py) and out of scope")
    _check_engine_config(config)
    if model_type == "gimmvfi_r":
        return GIMMVFI_R(config), None
    if model_type == "gimm":
        from .gimm import GIMM

        return GIMM(config), None
    if model_type == "gimmvfi_f":   # GIMM-VFI-F / F-P: native FlowFormer estimator + synthesis half (model_f.py)
        from .model_f import GIMMVFI_F

        return GIMMVFI_F(config), None
    raise ValueError("%s is not built in gimmvfi_b200 (gimmvfi_r, gimmvfi_f, gimm; see DESIGN.md scope)" % model_type)
