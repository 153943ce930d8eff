"""The drop-in modules' shared engine binding (gimmvfi_b200/module.py) on the H100: weights loaded into a submodule reach the engine
(the module then computes what a fresh module with the same full state_dict computes), and model.tensor_cores set between calls takes
effect.  The estimator outputs (raft_flow, nflow, the RAFT / FlowFormer flows) are deterministic and compared bit for bit; GIMM's
normalised flow passes through the softsplat's float atomics and is compared within 1e-5, in fp32."""
import pytest
import torch

import gimmvfi_r_oracle as O
from gimmvfi_b200 import GIMM, GIMMVFI_F, GIMMVFI_R, RAFT, FlowFormer
from gimmvfi_b200.synth import synth_batch, synth_flow_pair
from gimmvfi_b200.weights import random_state_dict, random_state_dict_f

pytestmark = pytest.mark.gpu
DEV = "cuda"
H, W = 128, 160


def subtree(sd, prefix):
    return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}


def interpolate(m, xs):
    """GIMMVFI_R / GIMMVFI_F at t = 0.5 -> its deterministic outputs"""
    o = m(xs, [(m.sample_coord_input(1, (H, W), [0.5], device=DEV), None)], t=[0.5 * torch.ones(1, device=DEV)])
    return o["raft_flow"], o["nflow"]


def estimate(m, xs):
    """RAFT / FlowFormer -> flow_up"""
    return m(255 * xs[:, :, 0], 255 * xs[:, :, 1])[0],


# module, the submodule a checkpoint is loaded into, that checkpoint (seed-1 weights), and the call whose outputs are compared
CASES = {
    "GIMMVFI_R": (GIMMVFI_R, "flow_estimator", lambda: subtree(random_state_dict(1), "flow_estimator."), interpolate),
    "GIMMVFI_F": (GIMMVFI_F, "flow_estimator", lambda: subtree(random_state_dict_f(1), "flow_estimator."), interpolate),
    "RAFT": (RAFT, "fnet", lambda: subtree(random_state_dict(1), "flow_estimator.fnet."), estimate),
    "FlowFormer": (FlowFormer, "memory_decoder", lambda: subtree(random_state_dict_f(1), "flow_estimator.memory_decoder."), estimate),
}


@pytest.mark.parametrize("name", list(CASES))
def test_checkpoint_loaded_into_a_submodule_reaches_the_engine(name):
    cls, sub, checkpoint, run = CASES[name]
    xs = synth_batch(1, H, W, seed=5).to(DEV)
    m = cls().to(DEV).eval()
    before = run(m, xs)
    m.get_submodule(sub).load_state_dict(checkpoint(), strict=True)
    after = run(m, xs)
    fresh = cls().to(DEV).eval()
    fresh.load_state_dict(m.state_dict(), strict=True)
    want = run(fresh, xs)
    for a, b, w in zip(before, after, want):
        assert torch.equal(b, w)
        assert not torch.equal(a, w)   # the new weights change the result: the comparison above is not vacuous


def test_gimm_checkpoint_loaded_into_hyponet_reaches_the_engine():
    B, h, w = 1, 64, 96
    ori = synth_flow_pair(B, h, w, seed=3)
    xs, _ = O.normalize_flow(ori)
    xs, ori = xs.to(DEV), ori.to(DEV)
    run = lambda m: m(xs, m.sample_coord_input(B, (h, w), [0.5], device=DEV), True, ori, 0.5 * torch.ones(B, device=DEV))
    m = GIMM().to(DEV).eval()
    m.tensor_cores = 0   # fp32: the atomics' jitter stays ~1e-7 (the TF32 HypoNet of the default mode amplifies it to ~5e-5)
    before = run(m)
    m.hyponet.load_state_dict(subtree(random_state_dict(1), "hyponet."), strict=True)
    after = run(m)
    fresh = GIMM().to(DEV).eval()
    fresh.tensor_cores = 0
    fresh.load_state_dict(m.state_dict(), strict=True)
    want = run(fresh)
    assert (after - want).abs().max().item() <= 1e-5
    assert (before - want).abs().max().item() > 1e-3


@pytest.mark.parametrize("name", ["GIMMVFI_R", "RAFT"])
def test_tensor_cores_set_between_calls_takes_effect(name):
    """the default mode, then fp32 on the same module: the second call equals a fresh module's fp32 call"""
    cls, _, _, run = CASES[name]
    xs = synth_batch(1, H, W, seed=5).to(DEV)
    m = cls().to(DEV).eval()
    default = run(m, xs)[0]
    m.tensor_cores = 0
    fp32 = run(m, xs)[0]
    fresh = cls().to(DEV).eval()
    fresh.tensor_cores = 0
    assert torch.equal(fp32, run(fresh, xs)[0])
    assert not torch.equal(default, fp32)
