"""LPIPS (Zhang et al., CVPR 2018) as the reference's evaluation drivers build it: ``LPIPS(net="alex", version="0.1")`` of
src/utils/lpips/lpips.py and ``calc_lpips`` of src/utils/lpips/__init__.py, computed by the native engine (AlexNet features on the
wgmma tensor cores in the fp32-class 3xF16 form, the calibrated head as CUDA kernels).  No torchvision and no download: the AlexNet
weights come from torchvision's own ``alexnet-owt-*.pth`` file, the calibration from the reference's ``alex.pth``."""
import os
from typing import Optional

import torch
import torch.nn as nn

from .module import EngineModule

CHANNELS = (64, 192, 384, 256, 256)
# torchvision AlexNet `features` index -> the LPIPS module's key (pretrained_networks.py:70-110 slices features[0:12] into 5 slices)
ALEX_TO_LPIPS = {0: "net.slice1.0", 3: "net.slice2.3", 6: "net.slice3.6", 8: "net.slice4.8", 10: "net.slice5.10"}
SHIFT = (-0.030, -0.088, -0.188)   # ScalingLayer (lpips.py:192-201)
SCALE = (0.458, 0.448, 0.450)


def lpips_keys() -> list:
    """the 22 keys of ``LPIPS(net="alex", version="0.1").state_dict()``, in the reference module's order"""
    keys = ["scaling_layer.shift", "scaling_layer.scale"]
    for name in ALEX_TO_LPIPS.values():
        keys += [name + ".weight", name + ".bias"]
    keys += ["lin%d.model.1.weight" % k for k in range(5)]
    keys += ["lins.%d.model.1.weight" % k for k in range(5)]
    return keys


class _NetLinLayer(nn.Module):
    """NetLinLayer (lpips.py:204-216): Sequential(Dropout, Conv2d(C, 1, 1, bias=False)); only its weight is used at inference"""

    def __init__(self, chn: int):
        super().__init__()
        self.model = nn.Sequential(nn.Dropout(), nn.Conv2d(chn, 1, 1, bias=False))


class _ScalingLayer(nn.Module):
    def __init__(self):
        super().__init__()
        self.register_buffer("shift", torch.tensor(SHIFT)[None, :, None, None])
        self.register_buffer("scale", torch.tensor(SCALE)[None, :, None, None])


class _AlexFeatures(nn.Module):
    """the parameter tree of pretrained_networks.alexnet: slice1..5 holding torchvision's features[0:12] under their indices"""

    def __init__(self):
        super().__init__()
        shapes = {0: (3, 64, 11), 3: (64, 192, 5), 6: (192, 384, 3), 8: (384, 256, 3), 10: (256, 256, 3)}
        for idx, name in ALEX_TO_LPIPS.items():
            sl = name.split(".")[1]
            if not hasattr(self, sl):
                self.add_module(sl, nn.Sequential())
            cin, cout, k = shapes[idx]
            getattr(self, sl).add_module(str(idx), nn.Conv2d(cin, cout, k))
        for p in self.parameters():
            p.requires_grad = False


class LPIPS(EngineModule):
    """``LPIPS(net="alex", version="0.1")`` with the reference's state_dict (22 keys, see lpips_keys()) and forward.

    Only the configuration calc_lpips builds exists: net="alex", version="0.1", lpips=True, spatial=False; anything else raises
    NotImplementedError.  The weights are the module's state_dict (``load_state_dict(reference_module.state_dict(), strict=True)``
    or lpips_state_dict() / load_lpips() from torchvision's AlexNet file and the reference's alex.pth).  CUDA tensors only."""

    def __init__(self, net: str = "alex", version: str = "0.1", lpips: bool = True, spatial: bool = False):
        super().__init__(lpips=True)
        if net != "alex":
            raise NotImplementedError("LPIPS (gimmvfi_b200): only net='alex' is built (got %r)" % (net,))
        if version != "0.1":
            raise NotImplementedError("LPIPS (gimmvfi_b200): only version='0.1' is built (got %r)" % (version,))
        if not lpips:
            raise NotImplementedError("LPIPS (gimmvfi_b200): only lpips=True (the calibrated head) is built")
        if spatial:
            raise NotImplementedError("LPIPS (gimmvfi_b200): only spatial=False is built")
        self.scaling_layer = _ScalingLayer()
        self.net = _AlexFeatures()
        for k, c in enumerate(CHANNELS):
            self.add_module("lin%d" % k, _NetLinLayer(c))
        self.lins = nn.ModuleList([getattr(self, "lin%d" % k) for k in range(5)])   # the same modules, as lpips.py:91-97
        for p in self.parameters():
            p.requires_grad = False
        self.eval()
        self._track_loads()

    def _prepare(self, x: torch.Tensor, name: str) -> torch.Tensor:
        if not torch.is_tensor(x) or not x.is_cuda:
            raise RuntimeError("LPIPS (gimmvfi_b200): %s must be a CUDA tensor; there is no CPU path" % name)
        if x.device != self.scaling_layer.shift.device:
            raise RuntimeError("LPIPS (gimmvfi_b200): %s on %s, module on %s" % (name, x.device, self.scaling_layer.shift.device))
        return x.to(torch.float32).contiguous()

    def forward(self, in0: torch.Tensor, in1: torch.Tensor, retPerLayer: bool = False, normalize: bool = False, quantize: bool = False):
        """in0, in1 (N,3,H,W) in [-1,1] (or [0,1] with normalize=True) -> (N,1,1,1), as lpips.py:125-189.
        retPerLayer: also the list of the 5 layer terms, each (N,1,1,1).  quantize: calc_lpips's rounding to 8-bit levels first."""
        a, b = self._prepare(in0, "in0"), self._prepare(in1, "in1")
        with torch.no_grad():
            out, layers = self.engine.lpips_forward(a, b, normalize=normalize, quantize=quantize, per_layer=True)
        out = out.view(-1, 1, 1, 1)
        if retPerLayer:
            return out, [layers[:, k].reshape(-1, 1, 1, 1) for k in range(5)]
        return out


_CALC = {}


def calc_lpips(gt: torch.Tensor, out: torch.Tensor, model: Optional[LPIPS] = None) -> torch.Tensor:
    """utils/lpips/__init__.py:25-28: gt, out in [-1,1] -> LPIPS of the 8-bit quantised images with normalize=True, (N,1,1,1).
    The module is built once per device (set_calc_lpips_model) instead of on every call."""
    if model is None:
        dev = gt.device if torch.is_tensor(gt) else None
        model = _CALC.get(dev)
        if model is None:
            raise RuntimeError("calc_lpips: no LPIPS weights for %s; call set_calc_lpips_model(load_lpips(alexnet_path, lin_path)) "
                               "or pass model=" % (dev,))
    return model(gt, out, normalize=True, quantize=True)


def set_calc_lpips_model(model: LPIPS) -> LPIPS:
    """the module calc_lpips uses for tensors on its device"""
    _CALC[model.scaling_layer.shift.device] = model
    return model


def lpips_state_dict(alexnet_sd: dict, lin_sd: dict) -> dict:
    """torchvision's AlexNet state_dict (``features.{0,3,6,8,10}.{weight,bias}``; classifier keys are ignored) and the reference's
    alex.pth (``lin{0..4}.model.1.weight``) -> the 22-key LPIPS state_dict"""
    sd = {"scaling_layer.shift": torch.tensor(SHIFT)[None, :, None, None], "scaling_layer.scale": torch.tensor(SCALE)[None, :, None, None]}
    for idx, name in ALEX_TO_LPIPS.items():
        for leaf in ("weight", "bias"):
            key = "features.%d.%s" % (idx, leaf)
            if key not in alexnet_sd:
                raise KeyError("lpips_state_dict: the AlexNet state_dict has no '%s'" % key)
            sd["%s.%s" % (name, leaf)] = alexnet_sd[key].detach().to(torch.float32).cpu().clone()
    for k in range(5):
        key = "lin%d.model.1.weight" % k
        if key not in lin_sd:
            raise KeyError("lpips_state_dict: the LPIPS calibration has no '%s'" % key)
        w = lin_sd[key].detach().to(torch.float32).cpu().clone()
        if tuple(w.shape) != (1, CHANNELS[k], 1, 1):
            raise ValueError("lpips_state_dict: '%s' has shape %s, expected %s" % (key, tuple(w.shape), (1, CHANNELS[k], 1, 1)))
        sd[key] = w
        sd["lins.%d.model.1.weight" % k] = w
    return {k: sd[k] for k in lpips_keys()}


def load_lpips(alexnet_path: str, lin_path: str, device="cuda") -> LPIPS:
    """LPIPS from torchvision's ImageNet AlexNet file (alexnet-owt-*.pth, e.g. from the torch hub cache) and the reference's
    src/utils/lpips/alex.pth, on `device`"""
    for p, what in ((alexnet_path, "AlexNet weights"), (lin_path, "LPIPS calibration (alex.pth)")):
        if not p or not os.path.isfile(p):
            raise FileNotFoundError("load_lpips: %s file not found: %s" % (what, p))
    alex = torch.load(alexnet_path, map_location="cpu", weights_only=True)
    lin = torch.load(lin_path, map_location="cpu", weights_only=True)
    m = LPIPS()
    m.load_state_dict(lpips_state_dict(alex, lin), strict=True)
    return m.to(device)
