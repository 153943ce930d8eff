"""The drop-in modules' shared engine binding (gimmvfi_b200/module.py) without a GPU: each module's parameter tree is the one it had
before the binding was shared, a load into any submodule marks the engine's weights stale (in a deepcopy too), and every module
refuses the CPU."""
import copy
import functools
import hashlib

import pytest
import torch
import torch.nn as nn

from gimmvfi_b200 import GIMM, GIMMVFI_F, GIMMVFI_R, RAFT, FlowFormer
from gimmvfi_b200.lpips import LPIPS

MODULES = {"GIMMVFI_R": GIMMVFI_R, "GIMMVFI_F": GIMMVFI_F, "GIMM": GIMM, "RAFT": RAFT, "FlowFormer": FlowFormer, "LPIPS": LPIPS}


@functools.lru_cache(maxsize=None)
def module(name):
    return MODULES[name]()


def inventory(m: nn.Module) -> str:
    """One line per state_dict entry: key, shape, dtype, Parameter (with its requires_grad) or buffer, and the first key whose tensor
    has the same storage (the sharing group); then the names of named_modules()."""
    lines, groups = [], {}
    for k, v in m.state_dict(keep_vars=True).items():
        g = groups.setdefault(v.untyped_storage().data_ptr(), k)
        kind = "param grad=%d" % v.requires_grad if isinstance(v, nn.Parameter) else "buffer"
        lines.append("%s %s %s %s %s" % (k, tuple(v.shape), v.dtype, kind, g))
    lines += [n for n, _ in m.named_modules()]
    return "\n".join(lines)


# sha256 of inventory(cls()), taken with this function on the modules as they were before module.py existed, when each module built
# its own tree (the norm3 / downsample.1 and lin<k> / lins.<k> sharing included)
DIGESTS = {
    "GIMMVFI_R": "7d207af90585a15258c9da1dcad20ec533e12048e8aaa2969d150dc9862ad846",
    "GIMMVFI_F": "2e282e800d78a26c22723d4553b544ddd6d508cd02d4dc48b00ab33e1b34062c",
    "GIMM": "b070e5b80e69c5bafabb31d156597aff9b51c4afaf7579a03a94d7c27384fc94",
    "RAFT": "9c81bdc0835933eacd6f99e3c49fda1a13d681968e361228cb1918e4f076122e",
    "FlowFormer": "a27bf2d846cf5c13d03c9cb137dec2c4878913f83cbbc272aebe35344c36a2e6",
    "LPIPS": "b0c641e11c2612be50b75f11cca9dc125b00d4f7bc48b9395c5d8e39fbaf6f7b",
}


@pytest.mark.parametrize("name", list(MODULES))
def test_parameter_tree_is_unchanged(name):
    assert hashlib.sha256(inventory(module(name)).encode()).hexdigest() == DIGESTS[name]


SUBMODULE = {"GIMMVFI_R": "flow_estimator", "GIMMVFI_F": "flow_estimator", "GIMM": "hyponet", "RAFT": "fnet",
             "FlowFormer": "memory_decoder", "LPIPS": "net.slice1"}


@pytest.mark.parametrize("name", list(MODULES))
def test_every_load_marks_the_weights_stale(name):
    """a checkpoint loaded into a submodule (e.g. RAFT weights into GIMMVFI_R.flow_estimator) must reach the engine: the root's weights
    are stale afterwards, as after a load into the root and after .to()"""
    m = module(name)
    sub = m.get_submodule(SUBMODULE[name])
    loads = [lambda: sub.load_state_dict({k: v + 1 if v.is_floating_point() else v for k, v in sub.state_dict().items()}, strict=True),
             lambda: m.load_state_dict(m.state_dict(), strict=True),
             lambda: m.to("cpu")]
    for load in loads:
        m._weights_dirty = False
        load()
        assert m._weights_dirty


@pytest.mark.parametrize("name", list(MODULES))
def test_loads_into_a_deepcopy_mark_the_copy_stale(name):
    """a deepcopy's hooks refer to the copy: a load into the copy or into one of its submodules marks the copy's weights stale, and
    leaves the original's as they are"""
    m = module(name)
    c = copy.deepcopy(m)
    sub = c.get_submodule(SUBMODULE[name])
    for load in (lambda: c.load_state_dict(c.state_dict(), strict=True), lambda: sub.load_state_dict(sub.state_dict(), strict=True)):
        m._weights_dirty = c._weights_dirty = False
        load()
        assert c._weights_dirty and not m._weights_dirty
    if name == "GIMMVFI_R":
        assert c.flow_estimator.__dict__["_model"]() is c   # the copy's flow_estimator runs on the copy's engine


def _cpu_call(name, m):
    x = torch.zeros(1, 3, 128, 128)
    if name in ("GIMMVFI_R", "GIMMVFI_F"):
        return m(torch.zeros(1, 3, 2, 128, 128), [(torch.zeros(1, 1, 128, 128, 3), None)], t=[torch.ones(1) * 0.5])
    if name == "GIMM":
        return m(torch.zeros(1, 2, 2, 64, 64), torch.zeros(1, 1, 64, 64, 3), True, torch.zeros(1, 2, 2, 64, 64), torch.ones(1) * 0.5)
    return m(x, x)


@pytest.mark.parametrize("name", list(MODULES))
def test_no_cpu_fallback(name):
    m = module(name)
    with pytest.raises(RuntimeError, match="CUDA"):
        _cpu_call(name, m)
    with pytest.raises(RuntimeError, match="CUDA"):
        m.engine
    if name == "GIMMVFI_R":
        with pytest.raises(RuntimeError, match="CUDA"):
            m.flow_estimator(torch.zeros(1, 3, 128, 128), torch.zeros(1, 3, 128, 128))
