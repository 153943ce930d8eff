"""TEST INFRASTRUCTURE — generates the GIMM-VFI-R fixtures at frame sizes that are multiples of 8 but not of 32
(tests/golden/r8_*.npz + manifest_r8.json) by running the UNMODIFIED reference (through oracle/ref_shim.py) on seeded
synthetic inputs and seeded random weights.  Runs only in the build container.

    python oracle/make_golden_r8.py

At these sizes RAFT runs on an odd h/8 x w/8 grid, the correlation pyramid floors odd levels and every tile loop of the
engine ends on a ragged edge:
    136x200        RAFT 17x25, pyramid 17x25 -> 8x12 -> 4x6 -> 2x3, H/4 = 34x50
    2 x 128x136    RAFT 16x17 (w = 17), two timesteps
    272x400 ds 0.5 the network runs at 136x200

Same keys as oracle/make_golden.py (imgt_pred / flowt stored at full resolution: stride 1), plus the max |Δ| of the travelling
oracle (oracle/gimmvfi_r_oracle.py) against the reference on the same case.
"""
import json
import os
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
warnings.filterwarnings("ignore")

import gimmvfi_r_oracle as O  # noqa: E402
import golden  # noqa: E402
import ref_shim  # noqa: E402
from gimmvfi_b200.synth import synth_batch  # noqa: E402
from gimmvfi_b200.weights import random_state_dict  # noqa: E402

# name, B, H, W, timesteps, ds_factor, input seed, weight seed, spatial stride for storage
CASES = [
    ("r8_136x200_t0.5", 1, 136, 200, [0.5], None, 41, 0, 1),
    ("r8_b2_128x136_t0.25_0.75", 2, 128, 136, [0.25, 0.75], None, 42, 0, 1),
    ("r8_ds0.5_272x400_t0.5", 1, 272, 400, [0.5], 0.5, 43, 0, 1),
]


def sub(t, s):
    return t[..., ::s, ::s].contiguous().numpy()


def main():
    torch.set_grad_enabled(False)
    out_dir = os.path.join(ROOT, "tests", "golden")
    manifest = {}
    sd = random_state_dict(0)
    model = ref_shim.build_reference_model(sd)
    for name, B, H, W, ts, ds, iseed, wseed, stride in CASES:
        assert wseed == 0
        xs = synth_batch(B, H, W, seed=iseed)
        ratio = 1.0 if ds is None else ds
        coord = [(model.sample_coord_input(B, (H, W), [t], device=xs.device, upsample_ratio=ratio), None) for t in ts]
        tt = [t * torch.ones(B) for t in ts]
        ref = model(xs, coord, t=tt, ds_factor=ds)
        ora = O.gimmvfi_r_forward(sd, xs, [(O.sample_coord_input(B, (H, W), [t], ratio), None) for t in ts], tt, ds_factor=ds)
        pin = 0.0
        for k in ("imgt_pred", "flowt", "ninrflow"):
            for a, b in zip(ref[k], ora[k]):
                pin = max(pin, (a - b).abs().max().item())
        pin = max(pin, (ref["raft_flow"] - ora["raft_flow"]).abs().max().item())
        arrays = {"stride": np.int32(stride)}
        for i in range(len(ts)):
            arrays["imgt_pred_%d" % i] = sub(ref["imgt_pred"][i], stride)
            arrays["flowt_%d" % i] = sub(ref["flowt"][i], stride)
            arrays["img_warp_4_%d" % i] = sub(ref["other_pred"][i][0], stride * 2)
            arrays["flowt0_4_%d" % i] = sub(ref["flowt0_pred"][i][1], stride)
            arrays["imgt_pred_sum_%d" % i] = np.float64(ref["imgt_pred"][i].double().sum().item())
        arrays["raft_flow"] = sub(ref["raft_flow"], stride * 2)
        arrays["raft_flow_absmax"] = np.float32(ref["raft_flow"].abs().max().item())
        golden.save(out_dir, name, arrays)
        manifest[name] = dict(B=B, H=H, W=W, timesteps=ts, ds_factor=ds, input_seed=iseed, weight_seed=wseed,
                              stride=stride, oracle_vs_reference_max_abs=pin)
        print(name, "oracle-vs-reference max|Δ| =", pin, flush=True)
    with open(os.path.join(out_dir, "manifest_r8.json"), "w") as f:
        json.dump(manifest, f, indent=1)


if __name__ == "__main__":
    main()
