"""Which weights an engine holds, on the host simulation (tests/hostsim): every entry point serves exactly the weight sets that can run
it and names what is missing otherwise, a weight set loaded over another leaves nothing of the old one reachable, and with debug taps
on every forward runs inside the workspace its own plan asked for."""
import ctypes as C
import os
import sys

import pytest
import torch

import gimmvfi_r_oracle as O
from gimmvfi_b200._lib import FlowInputs, GimmvfiError, IO, Problem, view_of
from gimmvfi_b200.gimm import GIMM_KEY_PREFIXES
from gimmvfi_b200.lpips import LPIPS
from gimmvfi_b200.weights import random_state_dict_f

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim"))
from harness import hostsim_engine  # noqa: E402

FE = "flow_estimator."


@pytest.fixture(scope="module")
def weight_sets(weights0):
    """name of the set in refusals -> (state_dict, load_state_dict keyword)"""
    f = random_state_dict_f(0)
    torch.manual_seed(0)
    return {
        "GIMM-VFI-R": (weights0, {}),
        "GIMM-VFI-F": (f, dict(full_f=True)),
        "synthesis": (f, dict(synthesis_only=True)),
        "GIMM": ({k: v for k, v in weights0.items() if k.startswith(GIMM_KEY_PREFIXES)}, dict(gimm_only=True)),
        "RAFT": ({k[len(FE):]: v for k, v in weights0.items() if k.startswith(FE)}, dict(raft=True)),
        "FlowFormer": ({k[len(FE):]: v for k, v in f.items() if k.startswith(FE)}, dict(flowformer=True)),
        "LPIPS": (LPIPS().state_dict(), dict(lpips=True)),
    }


@pytest.fixture(scope="module")
def engines(weight_sets):
    out = {}
    for name, (sd, kw) in weight_sets.items():
        out[name] = hostsim_engine()
        out[name].load_state_dict(sd, **kw)
    return out


def op_hyponet(e):
    """HypoNet on a 1 x 8 x 8 latent queried on a 12 x 12 grid (the resampling fp32-class form)"""
    lat = torch.zeros(1, 8, 8, 32)
    coord = O.sample_coord_input(1, (8, 8), [0.5], 1.5).contiguous()
    out = torch.empty(1, coord.shape[2], coord.shape[3], 2)
    e.lib.check(e.lib.dll.gimmvfi_op_hyponet(e._h, C.byref(view_of(lat)), C.c_void_p(coord.data_ptr()), C.byref(view_of(out)), 1, None), e._h)


def size_t():
    return C.byref(C.c_size_t())


def P(B, H, W, T=1):
    return C.byref(Problem(B, H, W, T, 0.0, H, W))


# entry point -> (the weight sets that serve it, what a refusal names as missing, a call).  The forwards get null pointers: an engine
# that serves one gets as far as its argument check, so the weight check must come first.
NULL = [None] * 8
ENTRIES = {
    "plan": ({"GIMM-VFI-R", "GIMM-VFI-F"}, "GIMM-VFI-R or GIMM-VFI-F", lambda d, h: d.gimmvfi_plan(h, P(1, 128, 128), size_t())),
    "forward": ({"GIMM-VFI-R", "GIMM-VFI-F"}, "GIMM-VFI-R or GIMM-VFI-F",
                lambda d, h: d.gimmvfi_forward(h, P(1, 64, 64), C.byref(IO()), None, 0, None)),
    "plan_from_flow": ({"GIMM-VFI-R", "GIMM-VFI-F", "synthesis"}, "synthesis", lambda d, h: d.gimmvfi_plan_from_flow(h, P(1, 128, 128), size_t())),
    "forward_from_flow": ({"GIMM-VFI-R", "GIMM-VFI-F", "synthesis"}, "synthesis",
                          lambda d, h: d.gimmvfi_forward_from_flow(h, P(1, 64, 64), C.byref(IO()), C.byref(FlowInputs()), None, 0, None)),
    "plan_gimm": ({"GIMM-VFI-R", "GIMM-VFI-F", "synthesis", "GIMM"}, "GIMM", lambda d, h: d.gimmvfi_gimm_plan(h, P(1, 40, 56, 2), size_t())),
    "forward_gimm": ({"GIMM-VFI-R", "GIMM-VFI-F", "synthesis", "GIMM"}, "GIMM",
                     lambda d, h: d.gimmvfi_gimm_forward(h, P(1, 40, 56), *NULL[:5], None, 0, None)),
    "plan_raft": ({"GIMM-VFI-R", "RAFT"}, "RAFT", lambda d, h: d.gimmvfi_raft_plan(h, 2, 128, 128, 1, 0, size_t())),
    "forward_raft": ({"GIMM-VFI-R", "RAFT"}, "RAFT", lambda d, h: d.gimmvfi_raft_forward(h, None, 2, 64, 64, None, 1, 1, *NULL[:7], None, 0, None)),
    "plan_flowformer": ({"GIMM-VFI-F", "FlowFormer"}, "FlowFormer", lambda d, h: d.gimmvfi_flowformer_plan(h, 2, 64, 64, 1, size_t())),
    "forward_flowformer": ({"GIMM-VFI-F", "FlowFormer"}, "FlowFormer",
                           lambda d, h: d.gimmvfi_flowformer_forward(h, None, 2, 64, 64, None, 1, 1, 1, None, None, None, 0, None)),
    "plan_lpips": ({"LPIPS"}, "LPIPS", lambda d, h: d.gimmvfi_lpips_plan(h, 1, 64, 64, size_t())),
    "forward_lpips": ({"LPIPS"}, "LPIPS", lambda d, h: d.gimmvfi_lpips_forward(h, None, None, 1, 64, 64, 0, None, None, None, 0, None)),
}
HELD = {"GIMM-VFI-R": "finalize_weights)", "GIMM-VFI-F": "finalize_weights_f", "synthesis": "finalize_weights_synthesis", "GIMM": "finalize_weights_gimm",
        "RAFT": "finalize_weights_raft", "FlowFormer": "finalize_weights_flowformer", "LPIPS": "finalize_weights_lpips"}


@pytest.mark.parametrize("entry", sorted(ENTRIES))
def test_each_entry_point_serves_its_weight_sets(engines, entry):
    served, needs, call = ENTRIES[entry]
    for held, e in engines.items():
        rc = call(e.lib.dll, e._h)
        msg = e.lib.dll.gimmvfi_last_error(e._h).decode() if rc else ""
        if held in served:
            assert rc == 0 or "required" in msg, (entry, held, msg)
        else:
            assert rc != 0, (entry, held)
            assert "no %s weights were loaded" % needs in msg and "holds %s weights only" % held in msg and HELD[held] in msg, (entry, held, msg)


def test_hyponet_op_serves_the_weight_sets_holding_gimm(engines):
    for held, e in engines.items():
        if held in ENTRIES["forward_gimm"][0]:
            op_hyponet(e)
        else:
            with pytest.raises(GimmvfiError, match="no GIMM weights were loaded"):
                op_hyponet(e)


@pytest.mark.parametrize("other", ["LPIPS", "RAFT", "FlowFormer"])
def test_hyponet_op_refused_after_the_gimm_weights_are_replaced(weight_sets, other):
    """the HypoNet parameters of the first load are freed by the second: the op must not reach them"""
    e = hostsim_engine()
    for name in ("GIMM", other):
        sd, kw = weight_sets[name]
        e.load_state_dict(sd, **kw)
        if name == "GIMM":
            op_hyponet(e)
    with pytest.raises(GimmvfiError, match="no GIMM weights were loaded"):
        op_hyponet(e)


def test_debug_forwards_run_inside_their_plans(engines):
    """with debug taps on, the plans hold the snapshots the forwards keep (per-timestep GIMM regions, RAFT / FlowFormer tap copies)"""
    g = torch.Generator().manual_seed(0)
    r, ff = engines["GIMM-VFI-R"], engines["FlowFormer"]
    for e in (r, ff):
        e.set_debug(True)
    try:
        B, H, W, ts = 1, 40, 56, (0.25, 0.75)
        ori = 4 * torch.rand(B, 2, 2, H, W, generator=g) - 2
        xs, _ = O.normalize_flow(ori)
        coords = torch.stack([O.sample_coord_input(B, (H, W), [t], 1.0) for t in ts], 0).contiguous()
        out = r.gimm_forward(xs.contiguous(), ori.contiguous(), coords, torch.stack([t * torch.ones(B) for t in ts], 0).contiguous())
        assert out.shape == (2, B, 2, 1, H, W) and torch.isfinite(r.tap("gimm.latent")).all()
        o = r.raft_forward(255 * torch.rand(2, 3, 128, 128, generator=g), [(0, 1)], iters=2)
        assert o["flow_up"].shape == (1, 2, 128, 128) and r.tap("raft.corr_it0").shape == (1, 16, 16, 324)
        up = ff.flowformer_forward(255 * torch.rand(2, 3, 64, 64, generator=g), [(0, 1), (1, 0)], iters=1)
        assert up.shape == (2, 2, 64, 64) and torch.isfinite(ff.tap("ff.dec_corr_0")).all()
    finally:
        for e in (r, ff):
            e.set_debug(False)


def test_conflicting_weight_sets_are_refused():
    with pytest.raises(ValueError, match="lpips and raft"):
        hostsim_engine().load_state_dict({}, raft=True, lpips=True)
