"""EngineHandle: owns one native engine (one per GPU / host thread), the packed
weights and a cached workspace; turns torch tensors into the raw pointers of the
C ABI (include/gimmvfi_b200.h).  PyTorch is used for device memory and streams only."""
import contextlib
import ctypes as C
from typing import Dict, Optional

import torch

from ._lib import IO, Clip, FlowInputs, Lib, Problem, Queries, View, default_lib


# The auxiliary outputs of GIMMVFI_R / GIMMVFI_F.forward: key of the returned dict -> the engine outputs it is made of
AUX_OUTPUTS = {
    "other_pred": ("img_warp_4",), "flowt0_pred": ("flowt0_1", "flowt0_4"), "flowt1_pred": ("flowt1_1", "flowt1_4"),
    "raft_flow": ("raft_flow",), "ninrflow": ("ninrflow",), "nflow": ("nflow",), "flowt": ("flowt",),
}
_ENGINE_AUX = tuple(f for fs in AUX_OUTPUTS.values() for f in fs)


def aux_keys(sel) -> tuple:
    """model.aux_outputs -> the auxiliary keys it selects, in AUX_OUTPUTS order: True = all, False / None = none, or a collection
    of keys of the returned dict such as ("flowt",)"""
    if sel is None or isinstance(sel, (bool, int)):
        return tuple(AUX_OUTPUTS) if sel else ()
    keys = (sel,) if isinstance(sel, str) else tuple(sel)
    bad = [k for k in keys if k not in AUX_OUTPUTS]
    if bad:
        raise ValueError("aux_outputs: unknown output(s) %s; choose from %s" % (bad, list(AUX_OUTPUTS)))
    return tuple(k for k in AUX_OUTPUTS if k in keys)


def model_outputs(o: Dict[str, torch.Tensor], T: int, keys) -> dict:
    """the dict GIMMVFI_R / GIMMVFI_F.forward return (gimmvfi_r.py:370-407): imgt_pred plus the selected auxiliary keys"""
    out = {"imgt_pred": [o["imgt_pred"][i] for i in range(T)]}
    make = {
        "other_pred": lambda: [[o["img_warp_4"][i]] for i in range(T)],
        "flowt0_pred": lambda: [[o["flowt0_1"][i], o["flowt0_4"][i]] for i in range(T)],
        "flowt1_pred": lambda: [[o["flowt1_1"][i], o["flowt1_4"][i]] for i in range(T)],
        "raft_flow": lambda: o["raft_flow"],
        "ninrflow": lambda: [o["ninrflow"][i] for i in range(T)],
        "nflow": lambda: o["nflow"],
        "flowt": lambda: [o["flowt"][i].squeeze() for i in range(T)],  # .squeeze() as gimmvfi_r.py:370
    }
    out.update({k: make[k]() for k in keys})
    return out


class EngineHandle:
    def __init__(self, device, lib: Optional[Lib] = None, allow_hostsim: bool = False):
        self.lib = lib if lib is not None else default_lib()
        self.device = torch.device(device)
        info = self.lib.build_info()
        self.hostsim = "HOSTSIM" in info
        if self.hostsim and not allow_hostsim:
            raise RuntimeError("gimmvfi_b200: refusing to run the test-only host simulation as a product path")
        if not self.hostsim and self.device.type != "cuda":
            raise RuntimeError("gimmvfi_b200 runs on CUDA devices only (got %s); there is no CPU fallback" % self.device)
        h = C.c_void_p()
        idx = self.device.index if self.device.type == "cuda" and self.device.index is not None else 0
        if self.device.type == "cuda":
            idx = torch.cuda.current_device() if self.device.index is None else self.device.index
        self.lib.check(self.lib.dll.gimmvfi_create(idx, C.byref(h)))
        self._h = h
        self._index = idx
        if self.device.type == "cuda":
            self.device = torch.device("cuda", idx)
        self._ws = None
        self._plans: Dict[tuple, int] = {}
        # static_outputs: forward() returns the same output tensors on every call of a problem shape (overwritten by the next call) -
        # with set_cuda_graph(True) and caller-owned input tensors this makes every pointer repeat, i.e. every forward a graph replay
        self.static_outputs = False
        self._static = None

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                self.lib.dll.gimmvfi_destroy(self._h)
                self._h = None
        except Exception:
            pass

    # ------------------------------------------------------------------ weights
    _FINALIZE = {"gimm_only": "gimmvfi_finalize_weights_gimm", "synthesis_only": "gimmvfi_finalize_weights_synthesis",
                 "full_f": "gimmvfi_finalize_weights_f", "lpips": "gimmvfi_finalize_weights_lpips",
                 "flowformer": "gimmvfi_finalize_weights_flowformer", "raft": "gimmvfi_finalize_weights_raft"}

    def load_state_dict(self, sd: Dict[str, torch.Tensor], gimm_only: bool = False, synthesis_only: bool = False, full_f: bool = False,
                        lpips: bool = False, flowformer: bool = False, raft: bool = False):
        """gimm_only: `sd` is a standalone GIMM checkpoint (gimm.py's module tree), only gimm_forward() is available.
        synthesis_only: `sd` is a GIMM-VFI-F state_dict; its `flow_estimator.*` (FlowFormer) entries are skipped and only
        forward_from_flow() is available.
        full_f: `sd` is a complete GIMM-VFI-F state_dict: forward() runs the native FlowFormer estimator + the synthesis half.
        lpips: `sd` is the 22-key state_dict of LPIPS(net="alex", version="0.1"); only lpips_forward() is available.
        flowformer: `sd` is the FlowFormer module's state_dict (GIMM-VFI-F's flow_estimator.*, prefix stripped or not); only
        flowformer_forward() is available (a full_f engine serves it too).
        raft: `sd` is the RAFT module's state_dict (GIMM-VFI-R's flow_estimator.*, prefix stripped); only raft_forward() is available
        (a full GIMM-VFI-R engine serves it too).
        None of them: `sd` is a complete GIMM-VFI-R state_dict.  At most one may be set."""
        chosen = [k for k, on in dict(gimm_only=gimm_only, synthesis_only=synthesis_only, full_f=full_f, lpips=lpips, flowformer=flowformer,
                                      raft=raft).items() if on]
        if len(chosen) > 1:
            raise ValueError("load_state_dict: %s select different weight sets; set at most one" % " and ".join(chosen))
        fin = getattr(self.lib.dll, self._FINALIZE[chosen[0]] if chosen else "gimmvfi_finalize_weights")
        for k, v in sd.items():
            if not v.dtype.is_floating_point:
                continue  # num_batches_tracked
            if synthesis_only and k.startswith("flow_estimator."):
                continue
            t = v.detach().to("cpu", torch.float32).contiguous()
            shape = (C.c_int64 * max(t.dim(), 1))(*t.shape)
            self.lib.check(self.lib.dll.gimmvfi_load_weight(self._h, k.encode(), C.c_void_p(t.data_ptr()), shape, t.dim()), self._h)
        self.lib.check(fin(self._h), self._h)

    def set_debug(self, on: bool):
        self.lib.check(self.lib.dll.gimmvfi_set_debug(self._h, int(on)), self._h)
        self._plans.clear()

    def set_tensor_cores(self, mode: int):
        """0: fp32 CUDA cores; 1: post-RAFT convs on wgmma TF32; 2: + RAFT convs on wgmma 3xTF32; 3: + the final decoder's
        residual trunk stored in fp16 on wgmma f16 (conv_tc.cu); 4 (experimental): + the 32/64-channel full-resolution chains in
        fp16.  The workspace plan depends on the mode."""
        self.lib.check(self.lib.dll.gimmvfi_set_tensor_cores(self._h, int(mode)), self._h)
        self.tensor_cores = int(mode)
        self._plans.clear()

    FWARP_MODES = {"linear": 0, "softmax": 1, "sum": 2}         # GIMMVFI_FWARP_*
    ACTIVATIONS = {"siren": 0, "relu": 1, "silu": 2, "damp": 3}   # GIMMVFI_ACT_*

    def set_motion_config(self, fwarp_type: str = "linear", activation: str = "siren", w0: float = 1.0, output_bias: float = 0.5,
                          normalize_weight: bool = True):
        """GIMM's motion settings (the reference's fwarp_type and hyponet.activation / output_bias / normalize_weight); they take effect
        at the next load_state_dict and hold until another call.  The defaults are the shipped configs'."""
        if fwarp_type not in self.FWARP_MODES:
            raise ValueError("fwarp_type %r: choose from %s" % (fwarp_type, list(self.FWARP_MODES)))
        if activation not in self.ACTIVATIONS:
            raise ValueError("activation %r: choose from %s" % (activation, list(self.ACTIVATIONS)))
        self.lib.check(self.lib.dll.gimmvfi_set_motion_config(self._h, self.FWARP_MODES[fwarp_type], self.ACTIVATIONS[activation], float(w0),
                                                              float(output_bias), int(bool(normalize_weight))), self._h)

    def set_cuda_graph(self, on: bool):
        """Replay forward() from a recorded CUDA graph whenever problem, tensors (same addresses), stream and mode repeat; see
        include/gimmvfi_b200.h.  Callers that want replays keep their input / coordinate tensors alive and let outputs recycle."""
        self.lib.check(self.lib.dll.gimmvfi_set_cuda_graph(self._h, int(on)), self._h)

    @property
    def graph_replays(self) -> int:
        return int(self.lib.dll.gimmvfi_graph_replays(self._h))

    def set_profile(self, on: bool):
        self.lib.check(self.lib.dll.gimmvfi_set_profile(self._h, int(on)), self._h)

    def profile(self) -> dict:
        """Per-kernel CUDA-event totals of the last forward (set_profile(True) first)."""
        import json

        return json.loads(self.lib.dll.gimmvfi_profile_json(self._h, self._stream()).decode())

    def set_raft_iters(self, iters: int):
        self.lib.check(self.lib.dll.gimmvfi_set_raft_iters(self._h, int(iters)), self._h)

    def set_flowformer_iters(self, iters: int):
        """decoder_depth of the native FlowFormer memory decoder (default 32)"""
        self.lib.check(self.lib.dll.gimmvfi_set_flowformer_iters(self._h, int(iters)), self._h)

    @property
    def last_launches(self) -> int:
        return int(self.lib.dll.gimmvfi_last_launches(self._h))

    @property
    def weights_version(self) -> int:
        return int(self.lib.dll.gimmvfi_weights_version(self._h))

    def _check_inputs(self, *tensors):
        """contiguous fp32 on THIS engine's device (a tensor of another GPU would hand the kernels a foreign pointer)"""
        for x in tensors:
            if x.dtype != torch.float32 or not x.is_contiguous():
                raise RuntimeError("gimmvfi_b200: inputs must be contiguous float32 tensors")
            if x.device.type != self.device.type or (self.device.type == "cuda" and x.device.index != self._index):
                raise RuntimeError("gimmvfi_b200: input on %s, engine on %s:%d" % (x.device, self.device.type, self._index))

    def _guard(self):
        """torch's current device = the engine's for the duration of a call (stream lookup, torch.empty)"""
        return torch.cuda.device(self._index) if self.device.type == "cuda" else contextlib.nullcontext()

    def _stream(self) -> C.c_void_p:
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream if self.device.type == "cuda" else None)

    def _plan(self, key, plan_call) -> int:
        """workspace bytes of the call that key identifies: plan_call(size_t*) calls the plan export, once per key"""
        if key not in self._plans:
            n = C.c_size_t()
            self.lib.check(plan_call(C.byref(n)), self._h)
            self._plans[key] = int(n.value)
        return self._plans[key]

    def _workspace(self, nbytes: int) -> torch.Tensor:
        """the engine's workspace, grown to at least nbytes"""
        if self._ws is None or self._ws.numel() < nbytes:
            self._ws = None
            self._ws = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        return self._ws

    # ------------------------------------------------------------------ forward
    def _problem(self, B, Hf, Wf, T, ds, Hc, Wc) -> Problem:
        return Problem(B, Hf, Wf, T, float(ds) if ds else 0.0, Hc, Wc)

    def workspace_bytes(self, B, Hf, Wf, T, ds, Hc, Wc, from_flow: bool = False) -> int:
        key = (B, Hf, Wf, T, float(ds) if ds else 0.0, Hc, Wc)
        plan = self.lib.dll.gimmvfi_plan_from_flow if from_flow else self.lib.dll.gimmvfi_plan
        return self._plan(key + (bool(from_flow),), lambda n: plan(self._h, C.byref(self._problem(*key)), n))

    def frame_cache_bytes(self, B, Hf, Wf, T, ds, Hc, Wc) -> int:
        p = self._problem(B, Hf, Wf, T, ds, Hc, Wc)
        return int(self.lib.dll.gimmvfi_frame_cache_bytes(C.byref(p)))

    def forward(self, img_xs: torch.Tensor, coords: torch.Tensor, t: torch.Tensor, ds: Optional[float] = None,
                aux_outputs=True, frame_cache=None, flow_inputs=None) -> Dict[str, torch.Tensor]:
        """img_xs (B,3,2,Hf,Wf), coords (T,B,1,Hc,Wc,3), t (T,B): contiguous fp32 on self.device.
        aux_outputs: True = every output, False = imgt_pred only, or a collection of the engine outputs wanted besides imgt_pred
        (names of gimmvfi_io, e.g. ("flowt",)); only those are allocated and written.
        frame_cache = (uint8 device tensor of frame_cache_bytes(), load, store): see gimmvfi_set_frame_cache.
        flow_inputs = dict(flows (B,2,2,H,W), feat4 [2 x (B,128,H/4,W/4)], feat8 [2 x (B,256,H/8,W/8)], fnet [2 x (B,256,H/8,W/8)]):
        the outputs of an external flow estimator at the network resolution -> gimmvfi_forward_from_flow (GIMM-VFI-F)."""
        self._check_inputs(img_xs, coords, t)
        if flow_inputs is not None:
            flow_inputs = {k: (v.to(torch.float32).contiguous() if torch.is_tensor(v) else [u.to(torch.float32).contiguous() for u in v])
                           for k, v in flow_inputs.items()}
            self._check_inputs(flow_inputs["flows"], *flow_inputs["feat4"], *flow_inputs["feat8"], *flow_inputs["fnet"])
        with self._guard():
            return self._forward(img_xs, coords, t, ds, aux_outputs, frame_cache, flow_inputs)

    def _forward(self, img_xs, coords, t, ds, aux_outputs, frame_cache, flow_inputs=None):
        B, _, _, Hf, Wf = img_xs.shape
        T, _, _, Hc, Wc, _ = coords.shape
        H, W = (Hf, Wf) if not ds else (int(Hf * ds), int(Wf * ds))
        self._workspace(self.workspace_bytes(B, Hf, Wf, T, ds, Hc, Wc, from_flow=flow_inputs is not None))
        E = lambda *s: torch.empty(*s, dtype=torch.float32, device=self.device)
        aux = self._engine_aux(aux_outputs)
        okey = (B, Hf, Wf, T, float(ds) if ds else 0.0, Hc, Wc, aux)
        if self.static_outputs and self._static is not None and self._static[0] == okey:
            out = self._static[1]   # the SAME tensors as the previous call (aliasing is the caller's choice: static_outputs = True)
            return self._launch(out, img_xs, coords, t, B, Hf, Wf, T, ds, Hc, Wc, frame_cache, flow_inputs)
        out = {"imgt_pred": E(T, B, 3, Hf, Wf)}
        if flow_inputs is not None:
            fi = flow_inputs
            assert tuple(fi["flows"].shape) == (B, 2, 2, H, W), (tuple(fi["flows"].shape), (B, 2, 2, H, W))
            for j in range(2):
                assert tuple(fi["feat4"][j].shape) == (B, 128, H // 4, W // 4) and tuple(fi["feat8"][j].shape) == (B, 256, H // 8, W // 8)
                assert tuple(fi["fnet"][j].shape) == (B, 256, H // 8, W // 8)
        shapes = self._output_shapes(B, Hf, Wf, T, H, W, Hc, Wc)
        out.update({f: E(*shapes[f]) for f in aux})
        if self.static_outputs:
            self._static = (okey, out)
        return self._launch(out, img_xs, coords, t, B, Hf, Wf, T, ds, Hc, Wc, frame_cache, flow_inputs)

    @staticmethod
    def _engine_aux(aux_outputs) -> tuple:
        """forward's aux_outputs -> the engine outputs written besides imgt_pred, in gimmvfi_io order"""
        if aux_outputs is None or isinstance(aux_outputs, (bool, int)):
            return _ENGINE_AUX if aux_outputs else ()
        bad = [f for f in aux_outputs if f not in _ENGINE_AUX]
        if bad:
            raise ValueError("aux_outputs: unknown engine output(s) %s" % bad)
        return tuple(f for f in _ENGINE_AUX if f in aux_outputs)

    @staticmethod
    def _output_shapes(B, Hf, Wf, T, H, W, Hc, Wc) -> dict:
        return dict(img_warp_4=(T, B, 3, H, W), flowt0_1=(T, B, 3, 2, Hf, Wf), flowt1_1=(T, B, 3, 2, Hf, Wf),
                    flowt0_4=(T, B, 2, H // 4, W // 4), flowt1_4=(T, B, 2, H // 4, W // 4), raft_flow=(B, 2, 2, H, W),
                    nflow=(B, 2, 2, H, W), ninrflow=(T, B, 2, 1, Hc, Wc), flowt=(T, B, 2, Hc, Wc))

    CLIP_PLANS = 16

    @staticmethod
    def _clip_struct(n_frames: int, pairs):
        """a gimmvfi_clip and the host pair array it points at (keep both alive for the call)"""
        pl = [(int(a), int(b)) for a, b in pairs]
        flat = (C.c_int32 * max(2 * len(pl), 1))(*[i for ab in pl for i in ab])
        return Clip(int(n_frames), len(pl), C.cast(flat, C.c_void_p)), flat

    def clip_workspace_bytes(self, n_frames, pairs, Hf, Wf, T, ds, Hc, Wc) -> int:
        """workspace bytes of forward_clip with this frame count and pair list (RAFT's all-pairs volumes grow with the pairs)"""
        pl = tuple((int(a), int(b)) for a, b in pairs)
        p = self._problem(len(pl), Hf, Wf, T, ds, Hc, Wc)
        c, flat = self._clip_struct(n_frames, pl)
        key = ("clip", int(n_frames), pl, Hf, Wf, T, float(ds) if ds else 0.0, Hc, Wc, self.weights_version)   # (R and F plan differently)
        if key in self._plans:
            self._plans[key] = self._plans.pop(key)   # (most recently used last)
        n = self._plan(key, lambda nb: self.lib.dll.gimmvfi_plan_clip(self._h, C.byref(p), C.byref(c), nb))
        # the plan depends on the pair list, so the cache keeps only the CLIP_PLANS most recent lists (a video loop reuses one per call size)
        clip_keys = [k for k in self._plans if k[0] == "clip"]
        for k in clip_keys[:max(0, len(clip_keys) - self.CLIP_PLANS)]:
            del self._plans[k]
        return n

    def forward_clip(self, frames: torch.Tensor, pairs, coords: torch.Tensor, t: torch.Tensor, ds: Optional[float] = None,
                     aux_outputs=True) -> Dict[str, torch.Tensor]:
        """A clip in one engine call (gimmvfi_forward_clip): frames (F,3,Hf,Wf) in [0,1], pairs [(src, tgt), ...] of frame indices,
        coords (T,P,1,Hc,Wc,3), t (T,P), contiguous fp32 on self.device.  Returns forward()'s dict with the pair axis in place of the
        batch axis: pair p's entries are forward()'s with B = 1 on (frames[src], frames[tgt])."""
        self._check_inputs(frames, coords, t)
        if frames.dim() != 4 or frames.shape[1] != 3:
            raise ValueError("clip: frames must be (F,3,H,W), got %s" % (tuple(frames.shape),))
        F, _, Hf, Wf = frames.shape
        pl = [(int(a), int(b)) for a, b in pairs]
        P = len(pl)
        if P < 1:
            raise ValueError("clip: at least one pair is required")
        bad = [ab for ab in pl if not (0 <= ab[0] < F and 0 <= ab[1] < F)]
        if bad:
            raise ValueError("clip: pair(s) %s index outside the %d frames" % (bad, F))
        if coords.dim() != 6 or coords.shape[1] != P or coords.shape[2] != 1 or coords.shape[5] != 3:
            raise ValueError("clip: coords must be (T,%d,1,Hc,Wc,3), got %s" % (P, tuple(coords.shape)))
        T, Hc, Wc = coords.shape[0], coords.shape[3], coords.shape[4]
        if tuple(t.shape) != (T, P):
            raise ValueError("clip: t must be (%d,%d), got %s" % (T, P, tuple(t.shape)))
        H, W = (Hf, Wf) if not ds else (int(Hf * ds), int(Wf * ds))
        aux = self._engine_aux(aux_outputs)
        with self._guard():
            self._workspace(self.clip_workspace_bytes(F, pl, Hf, Wf, T, ds, Hc, Wc))
            E = lambda *s: torch.empty(*s, dtype=torch.float32, device=self.device)
            shapes = self._output_shapes(P, Hf, Wf, T, H, W, Hc, Wc)
            out = {"imgt_pred": E(T, P, 3, Hf, Wf)}
            out.update({f: E(*shapes[f]) for f in aux})
            io = IO()
            io.img_xs, io.coords, io.t = frames.data_ptr(), coords.data_ptr(), t.data_ptr()
            for k, v in out.items():
                setattr(io, k, v.data_ptr())
            p = self._problem(P, Hf, Wf, T, ds, Hc, Wc)
            c, flat = self._clip_struct(F, pl)
            self.lib.check(self.lib.dll.gimmvfi_forward_clip(self._h, C.byref(p), C.byref(c), C.byref(io), C.c_void_p(self._ws.data_ptr()),
                                                             self._ws.numel(), self._stream()), self._h)
        return out

    @staticmethod
    def _queries_struct(n_frames: int, queries):
        """a gimmvfi_queries and the host arrays it points at (keep all three alive for the call)"""
        ql = [(int(a), int(b), float(t)) for a, b, t in queries]
        flat = (C.c_int32 * max(2 * len(ql), 1))(*[i for a, b, _ in ql for i in (a, b)])
        ts = (C.c_float * max(len(ql), 1))(*[t for _, _, t in ql])
        return Queries(int(n_frames), len(ql), C.cast(flat, C.c_void_p), C.cast(ts, C.c_void_p)), flat, ts

    @staticmethod
    def query_pairs(queries):
        """the distinct (src, tgt) pairs of a query list in first-appearance order, and each query's index among them"""
        pairs, index = {}, []
        for a, b, _ in queries:
            index.append(pairs.setdefault((int(a), int(b)), len(pairs)))
        return list(pairs), index

    def queries_workspace_bytes(self, n_frames, queries, Hf, Wf, ds, Hc, Wc) -> int:
        """workspace bytes of forward_queries with this frame count and query list.  The plan depends on the frame count, the distinct
        pairs and their timestep counts only: plans are cached on that structure (the CLIP_PLANS most recent ones)."""
        pairs, index = self.query_pairs(queries)
        counts = tuple(index.count(i) for i in range(len(pairs)))
        key = ("queries", int(n_frames), tuple(pairs), counts, Hf, Wf, float(ds) if ds else 0.0, Hc, Wc, self.weights_version)
        if key in self._plans:
            self._plans[key] = self._plans.pop(key)   # (most recently used last)
        # any query list of this structure plans alike: t = 0.5 throughout
        rep = [(a, b, 0.5) for (a, b), c in zip(pairs, counts) for _ in range(c)]
        p = self._problem(len(pairs), Hf, Wf, max(counts), ds, Hc, Wc)
        q, flat, ts = self._queries_struct(n_frames, rep)
        n = self._plan(key, lambda nb: self.lib.dll.gimmvfi_plan_queries(self._h, C.byref(p), C.byref(q), nb))
        qkeys = [k for k in self._plans if k[0] == "queries"]
        for k in qkeys[:max(0, len(qkeys) - self.CLIP_PLANS)]:
            del self._plans[k]
        return n

    def forward_queries(self, frames: torch.Tensor, queries, ds: Optional[float] = None, aux_outputs=True,
                        coord_range=(-1.0, 1.0)) -> Dict[str, torch.Tensor]:
        """A query list in one engine call (gimmvfi_forward_queries): frames (F,3,Hf,Wf) in [0,1] contiguous fp32 on self.device, queries
        [(src, tgt, t), ...] with t strictly inside (0, 1).  The queries of one (src, tgt) are that pair's timesteps; the engine makes
        the coordinates (sample_coord_input at the network resolution over coord_range) and t.  Returns the engine outputs: per-timestep
        ones (Q, ...) in query order, raft_flow / nflow (P,2,2,H,W) over the distinct pairs in first-appearance order (query_pairs)."""
        self._check_inputs(frames)
        if frames.dim() != 4 or frames.shape[1] != 3:
            raise ValueError("queries: frames must be (F,3,H,W), got %s" % (tuple(frames.shape),))
        F, _, Hf, Wf = frames.shape
        ql = [(int(a), int(b), float(t)) for a, b, t in queries]
        if not ql:
            raise ValueError("queries: at least one query is required")
        Q = len(ql)
        P = len(self.query_pairs(ql)[0])
        H, W = (Hf, Wf) if not ds else (int(Hf * ds), int(Wf * ds))
        aux = self._engine_aux(aux_outputs)
        with self._guard():
            self._workspace(self.queries_workspace_bytes(F, ql, Hf, Wf, ds, H, W))
            E = lambda *s: torch.empty(*s, dtype=torch.float32, device=self.device)
            shapes = self._output_shapes(P, Hf, Wf, 1, H, W, H, W)
            out = {"imgt_pred": E(Q, 3, Hf, Wf)}
            out.update({f: E(*shapes[f]) if f in ("raft_flow", "nflow") else E(Q, *shapes[f][2:]) for f in aux})
            io = IO()
            io.img_xs = frames.data_ptr()
            for k, v in out.items():
                setattr(io, k, v.data_ptr())
            p = self._problem(P, Hf, Wf, 1, ds, H, W)
            q, flat, ts = self._queries_struct(F, ql)
            self.lib.check(self.lib.dll.gimmvfi_set_coord_range(self._h, float(coord_range[0]), float(coord_range[1])), self._h)
            self.lib.check(self.lib.dll.gimmvfi_forward_queries(self._h, C.byref(p), C.byref(q), C.byref(io), C.c_void_p(self._ws.data_ptr()),
                                                                self._ws.numel(), self._stream()), self._h)
        return out

    def _launch(self, out, img_xs, coords, t, B, Hf, Wf, T, ds, Hc, Wc, frame_cache, flow_inputs):
        io = IO()
        io.img_xs, io.coords, io.t = img_xs.data_ptr(), coords.data_ptr(), t.data_ptr()
        for k, v in out.items():
            setattr(io, k, v.data_ptr())
        p = self._problem(B, Hf, Wf, T, ds, Hc, Wc)
        if frame_cache is not None:
            buf, load, store = frame_cache
            assert buf.dtype == torch.uint8 and buf.is_contiguous() and buf.device == self.device
            self.lib.check(self.lib.dll.gimmvfi_set_frame_cache(self._h, C.c_void_p(buf.data_ptr()), buf.numel(), int(load), int(store)), self._h)
        try:
            if flow_inputs is not None:
                f = FlowInputs()
                f.flows = flow_inputs["flows"].data_ptr()
                for j in range(2):
                    f.feat4[j], f.feat8[j], f.fnet[j] = (flow_inputs[k][j].data_ptr() for k in ("feat4", "feat8", "fnet"))
                self.lib.check(self.lib.dll.gimmvfi_forward_from_flow(self._h, C.byref(p), C.byref(io), C.byref(f), C.c_void_p(self._ws.data_ptr()),
                                                                      self._ws.numel(), self._stream()), self._h)
            else:
                self.lib.check(self.lib.dll.gimmvfi_forward(self._h, C.byref(p), C.byref(io), C.c_void_p(self._ws.data_ptr()),
                                                            self._ws.numel(), self._stream()), self._h)
        finally:
            if frame_cache is not None:
                self.lib.check(self.lib.dll.gimmvfi_set_frame_cache(self._h, None, 0, 0, 0), self._h)
        return out

    def gimm_forward(self, xs: torch.Tensor, ori_flow: torch.Tensor, coords: torch.Tensor, t: torch.Tensor) -> torch.Tensor:
        """GIMM.forward (gimm.py:129-214): xs, ori_flow (B,2,2,H,W), coords (T,B,1,Hc,Wc,3), t (T,B) -> (T,B,2,1,Hc,Wc).
        The coordinate grid may have any size: HypoNet resizes the latent to it (hyponet.py:86-90)."""
        self._check_inputs(xs, ori_flow, coords, t)
        with self._guard():
            return self._gimm_forward(xs, ori_flow, coords, t)

    def _gimm_forward(self, xs, ori_flow, coords, t):
        B, _, _, H, W = xs.shape
        T = coords.shape[0]
        if coords.dim() != 6 or tuple(coords.shape[1:3]) != (B, 1) or coords.shape[5] != 3:
            raise ValueError("gimm_forward: coords must be (T,B,1,Hc,Wc,3) with B = %d, got %s" % (B, tuple(coords.shape)))
        Hc, Wc = coords.shape[3], coords.shape[4]
        assert tuple(ori_flow.shape) == (B, 2, 2, H, W) and tuple(t.shape) == (T, B)
        p = self._problem(B, H, W, T, None, Hc, Wc)
        ws = self._workspace(self._plan(("gimm", B, H, W, T, Hc, Wc), lambda n: self.lib.dll.gimmvfi_gimm_plan(self._h, C.byref(p), n)))
        out = torch.empty(T, B, 2, 1, Hc, Wc, dtype=torch.float32, device=self.device)
        P = lambda x: C.c_void_p(x.data_ptr())
        self.lib.check(self.lib.dll.gimmvfi_gimm_forward(self._h, C.byref(p), P(xs), P(ori_flow), P(coords), P(t), P(out), P(ws),
                                                         ws.numel(), self._stream()), self._h)
        return out

    def lpips_forward(self, in0: torch.Tensor, in1: torch.Tensor, normalize: bool = False, quantize: bool = False, per_layer: bool = False):
        """LPIPS(net="alex", version="0.1").forward (lpips.py:125-189): in0, in1 (n,3,h,w) -> (n,) distances, and with per_layer also
        the (n,5) spatial means of the layer terms.  quantize: calc_lpips's rounding to 8-bit levels first (utils/lpips/__init__.py:20-28)."""
        self._check_inputs(in0, in1)
        if in0.dim() != 4 or in0.shape[1] != 3 or in0.shape != in1.shape:
            raise ValueError("lpips: in0 and in1 must both be (n,3,h,w), got %s and %s" % (tuple(in0.shape), tuple(in1.shape)))
        n, _, h, w = in0.shape
        with self._guard():
            ws = self._workspace(self._plan(("lpips", n, h, w), lambda nb: self.lib.dll.gimmvfi_lpips_plan(self._h, n, h, w, nb)))
            out = torch.empty(n, dtype=torch.float32, device=self.device)
            layers = torch.empty(n, 5, dtype=torch.float32, device=self.device) if per_layer else None
            P = lambda x: C.c_void_p(x.data_ptr() if x is not None else None)
            flags = (1 if normalize else 0) | (2 if quantize else 0)
            self.lib.check(self.lib.dll.gimmvfi_lpips_forward(self._h, P(in0), P(in1), n, h, w, flags, P(out), P(layers), P(ws),
                                                              ws.numel(), self._stream()), self._h)
        return (out, layers) if per_layer else out

    def flowformer_forward(self, frames: torch.Tensor, pairs, pairs_per_call: int = 1, iters: int = 0, flow_low: bool = False,
                           flow_init: Optional[torch.Tensor] = None, features: bool = False):
        """FlowFormer.forward (transformer.py:45-74) for every (source, target) pair of frame indices: frames (F,3,H,W) float32 in
        [0,255], H and W multiples of 32 -> flow_up (P,2,H,W) [and flow_low (P,2,H/8,W/8), the last iteration's coords1 - coords0].
        Consecutive pairs form reference calls of pairs_per_call pairs (see include/gimmvfi_b200.h); iters 0 = the engine's decoder depth.
        flow_init (P,2,H/8,W/8) optional: the warm start of each pair (decoder.py:265-267).  features: return_feat=True, the result is then
        (flows, [cfeat4 (P,128,H/4,W/4), cfeat8 (P,256,H/8,W/8)], ffeat (P,256,H/8,W/8)) with flows as without it; the features are those
        of each pair's source frame.
        Memory per pair: the cost volume and the GMA attention matrix, N^2 floats each with N = (H/8)(W/8) (12.8 MB each at 256x448,
        4.3 GB each at 1088x1920): bound P accordingly."""
        self._check_inputs(frames)
        if frames.dim() != 4 or frames.shape[1] != 3:
            raise ValueError("flowformer: frames must be (F,3,H,W), got %s" % (tuple(frames.shape),))
        pl = [(int(a), int(b)) for a, b in pairs]
        F, _, H, W = frames.shape
        P = len(pl)
        if flow_init is not None:
            flow_init = flow_init.to(torch.float32).contiguous()
            self._check_inputs(flow_init)
            if tuple(flow_init.shape) != (P, 2, H // 8, W // 8):
                raise ValueError("flowformer: flow_init must be (%d,2,%d,%d), got %s" % (P, H // 8, W // 8, tuple(flow_init.shape)))
        flat = (C.c_int32 * max(2 * P, 1))(*[i for ab in pl for i in ab])
        with self._guard():
            ws = self._workspace(self._plan(("flowformer", F, H, W, P), lambda nb: self.lib.dll.gimmvfi_flowformer_plan(self._h, F, H, W, P, nb)))
            E = lambda *s: torch.empty(*s, dtype=torch.float32, device=self.device)
            up = E(P, 2, H, W)
            low = E(P, 2, H // 8, W // 8) if flow_low else None
            c4, c8, ff = (E(P, 128, H // 4, W // 4), E(P, 256, H // 8, W // 8), E(P, 256, H // 8, W // 8)) if features else (None, None, None)
            Pt = lambda x: C.c_void_p(x.data_ptr() if x is not None else None)
            self.lib.check(self.lib.dll.gimmvfi_flowformer_forward_ex(self._h, Pt(frames), F, H, W, flat, P, int(pairs_per_call), int(iters),
                                                                      Pt(flow_init), Pt(up), Pt(low), Pt(c4), Pt(c8), Pt(ff), Pt(ws), ws.numel(),
                                                                      self._stream()), self._h)
        flows = (up, low) if flow_low else up
        return (flows, [c4, c8], ff) if features else flows

    RAFT_OUTPUTS = ("flow_up", "flow_low", "flow_iters", "feat4", "feat8", "fmap")

    def raft_forward(self, frames: torch.Tensor, pairs, iters: int = 12, flow_init: Optional[torch.Tensor] = None, outputs=("flow_up",)) -> dict:
        """RAFT.forward (raft/raft.py:100-169) for every (source, target) pair of frame indices: frames (F,3,H,W) float32 in [0,255], H and W
        multiples of 8 and >= 128; flow_init (P,2,H/8,W/8) optional.  outputs: the names wanted, of flow_up (P,2,H,W), flow_low
        (P,2,H/8,W/8), flow_iters (iters,P,2,H,W), feat4 (P,96,H/4,W/4), feat8 (P,128,H/8,W/8) and fmap (P,256,H/8,W/8) (see
        include/gimmvfi_b200.h) -> {name: tensor}.  Memory per pair: the volume pyramid, N^2 * 4/3 floats with N = (H/8)(W/8)."""
        self._check_inputs(frames)
        if frames.dim() != 4 or frames.shape[1] != 3:
            raise ValueError("raft: frames must be (F,3,H,W), got %s" % (tuple(frames.shape),))
        bad = [k for k in outputs if k not in self.RAFT_OUTPUTS]
        if bad:
            raise ValueError("raft: unknown output(s) %s; choose from %s" % (bad, list(self.RAFT_OUTPUTS)))
        pl = [(int(a), int(b)) for a, b in pairs]
        F, _, H, W = frames.shape
        P, iters = len(pl), int(iters)
        if flow_init is not None:
            flow_init = flow_init.to(torch.float32).contiguous()
            self._check_inputs(flow_init)
            if tuple(flow_init.shape) != (P, 2, H // 8, W // 8):
                raise ValueError("raft: flow_init must be (%d,2,%d,%d), got %s" % (P, H // 8, W // 8, tuple(flow_init.shape)))
        flat = (C.c_int32 * max(2 * P, 1))(*[i for ab in pl for i in ab])
        with self._guard():
            want_iters = "flow_iters" in outputs
            plan = lambda nb: self.lib.dll.gimmvfi_raft_plan(self._h, F, H, W, P, int(want_iters), nb)
            ws = self._workspace(self._plan(("raft", F, H, W, P, want_iters), plan))
            shapes = dict(flow_up=(P, 2, H, W), flow_low=(P, 2, H // 8, W // 8), flow_iters=(max(iters, 0), P, 2, H, W),
                          feat4=(P, 96, H // 4, W // 4), feat8=(P, 128, H // 8, W // 8), fmap=(P, 256, H // 8, W // 8))
            out = {k: torch.empty(*shapes[k], dtype=torch.float32, device=self.device) for k in self.RAFT_OUTPUTS if k in outputs}
            Pt = lambda x: C.c_void_p(x.data_ptr() if x is not None else None)
            self.lib.check(self.lib.dll.gimmvfi_raft_forward(self._h, Pt(frames), F, H, W, flat, P, iters, Pt(flow_init),
                                                             *[Pt(out.get(k)) for k in self.RAFT_OUTPUTS], Pt(ws), ws.numel(), self._stream()),
                           self._h)
        return out

    def tap(self, name: str) -> torch.Tensor:
        """Debug: copy of an intermediate NHWC tensor of the last forward (set_debug(True) first).
        Taps are read as float32: every tapped tensor is fp32 in all precision modes (the half-precision tensors of modes 3-4 that
        are tapped - syn.fup1, syn.fin1 - are fp32 snapshots of the stored half values).  The per-timestep taps (gimm.splat0 / splat1,
        gimm.latent, syn.* apart from syn.feat4 / feat8 / fup4 / fup1 / fproj) are taken at the LAST timestep, whose buffers nothing
        overwrites after it.  Every timestep depends only on the t-independent state and its own t / coordinates, so to inspect a
        timestep, put it last."""
        v = View()
        self.lib.check(self.lib.dll.gimmvfi_get_tap(self._h, name.encode(), C.byref(v)), self._h)
        base = self._ws.data_ptr()
        off = (v.data - base) // 4
        flat = self._ws.view(torch.float32)
        t = torch.as_strided(flat, (v.n, v.h, v.w, v.c), (v.batch_stride, v.w * v.pixel_stride, v.pixel_stride, 1), off)
        return t.clone()
