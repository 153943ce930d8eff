"""EngineModule: the base of every drop-in module that runs on the native engine (GIMMVFI_R, GIMMVFI_F, GIMM, RAFT, FlowFormer and
LPIPS).  It owns the module's EngineHandle, uploads the module's weights into it whenever they changed, and builds the reference's
parameter tree from a (key, shape, dtype) spec."""
import weakref
from typing import Optional

import torch
import torch.nn as nn

from .engine import EngineHandle


class _Node(nn.Module):
    """Anonymous container used to reproduce the reference's module tree names."""


def load_estimator_checkpoint(path_or_dict) -> dict:
    """initialize_RAFT's and initialize_Flowformer's convert (raft/__init__.py:16-19, flowformer/__init__.py): keep the keys containing
    "module" and drop "module." from them.  Takes a path (torch.load on the CPU, e.g. raft-things.pth or flowformer_sintel.pth, the
    checkpoints the estimators of GIMM-VFI-R and GIMM-VFI-F start from, configs/submission.py:17) or an already loaded dict."""
    ckpt = torch.load(path_or_dict, map_location="cpu") if isinstance(path_or_dict, str) else path_or_dict
    return {k.replace("module.", ""): v for k, v in ckpt.items() if "module" in k}


class _RootRef:
    """A weak reference to an EngineModule from inside its own tree (a strong one would be a reference cycle that keeps a dropped
    model's engine alive until the garbage collector runs).  In a deepcopy of the tree it refers to the copied root."""

    def __init__(self, root):
        self._ref = weakref.ref(root)

    def __call__(self):
        return self._ref()

    def __deepcopy__(self, memo):
        root = self._ref()
        root = memo.get(id(root), root)   # copy.deepcopy memoises the copied root before it copies the root's state
        return _RootRef(root) if root is not None else self


class _MarkStale:
    """load_state_dict post-hook of every module in an EngineModule's tree: marks the root's engine weights stale"""

    def __init__(self, root):
        self.root = _RootRef(root)

    def __call__(self, module, incompatible_keys):
        root = self.root()
        if root is not None:
            root._weights_dirty = True


class EngineModule(nn.Module):
    def __init__(self, **weight_set):
        """weight_set: the EngineHandle.load_state_dict keyword naming the module's weight set, e.g. raft=True; none = GIMM-VFI-R"""
        super().__init__()
        self._weight_set = weight_set
        self._engine: Optional[EngineHandle] = None
        self._weights_dirty = True

    def _track_loads(self):
        """Marks the engine's weights stale after a load_state_dict into this module or into any of its submodules, e.g. a RAFT
        checkpoint loaded into model.flow_estimator.  Called once the module tree is complete."""
        stale = _MarkStale(self)
        for m in self.modules():
            m.register_load_state_dict_post_hook(stale)

    def _apply(self, fn, *a, **k):
        r = super()._apply(fn, *a, **k)
        self._weights_dirty = True
        return r

    def refresh_weights(self):
        """Re-pack + upload the weights (automatic after load_state_dict / .to()).  The handle is kept while the device stays the
        same, so settings made on it (set_cuda_graph, set_raft_iters, static_outputs, ...) survive a reload."""
        dev = next(self.parameters()).device
        if dev.type != "cuda":
            raise RuntimeError("%s (gimmvfi_b200) runs on CUDA devices only; call .to('cuda') first, there is no CPU path" % type(self).__name__)
        if self._engine is None or self._engine.device != dev:
            self._engine = EngineHandle(dev)
        self._engine.load_state_dict(self.state_dict(), **self._weight_set)
        self._engine.tensor_cores = None
        self._weights_dirty = False

    @property
    def engine(self) -> EngineHandle:
        if self._engine is None or self._weights_dirty:
            self.refresh_weights()
        return self._engine

    def _ready(self, x: torch.Tensor) -> EngineHandle:
        """the engine for a call on input x: refuses a non-CUDA x, then applies self.tensor_cores (a module without one, LPIPS,
        leaves the engine's mode as it is)"""
        if x.device.type != "cuda":
            raise RuntimeError("%s (gimmvfi_b200): inputs must live on a CUDA device; there is no CPU path" % type(self).__name__)
        eng = self.engine
        tc = getattr(self, "tensor_cores", None)
        if tc is not None and getattr(eng, "tensor_cores", None) != int(tc):
            eng.set_tensor_cores(int(tc))
        return eng

    def build_params(self, spec, init, init_prefix: str = ""):
        """Registers every (key, shape, dtype) of `spec` under the module path its key names, initialised from init[init_prefix + key]:
        int64 entries, running_mean and running_var as buffers, the rest as Parameters without grad.  Missing containers are _Node;
        a container registered before the call is used as it is.  A `.downsample.1.` entry is its `.norm3.` twin's tensor: RAFT's
        residual blocks register norm3 under both names (raft/extractor.py:44-47)."""
        made = {}
        for key, _, dt in spec:
            *path, leaf = key.split(".")
            mod = self
            for p in path:
                if p not in mod._modules:
                    mod.add_module(p, _Node())
                mod = mod._modules[p]
            obj = made.get(key.replace(".downsample.1.", ".norm3."))   # None unless key is a downsample.1 entry
            if obj is None:
                t = init[init_prefix + key].clone()
                obj = t if dt == "int64" or leaf in ("running_mean", "running_var") else nn.Parameter(t, requires_grad=False)
            made[key] = obj
            if isinstance(obj, nn.Parameter):
                mod.register_parameter(leaf, obj)
            else:
                mod.register_buffer(leaf, obj)
        self._track_loads()
