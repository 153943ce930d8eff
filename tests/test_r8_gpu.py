"""End-to-end GPU parity of GIMMVFI_R at frame sizes that are multiples of 8 but not of 32, against fixtures of the unmodified
reference (oracle/make_golden_r8.py).  At these sizes RAFT runs on an odd h/8 x w/8 grid (17 x 25, 16 x 17), the correlation pyramid
floors odd levels, the FlowHead's four-pixel quads end on a partial quad and every tile loop ends on a ragged edge.

Same outputs, same bars as tests/test_forward_gpu.py (whose helpers run the model and do the comparison), in every precision mode
and on the volume-free RAFT lookup."""
import json
import os

import pytest

from conftest import GOLDEN_DIR
from gimmvfi_b200 import GIMMVFI_R
from golden import load as load_golden
from test_forward_gpu import golden_checks, model, report_checks  # noqa: F401  (`model`: the fixture over all precision modes)

pytestmark = pytest.mark.gpu
DEV = "cuda"
CASES = ["r8_136x200_t0.5", "r8_b2_128x136_t0.25_0.75", "r8_ds0.5_272x400_t0.5"]


@pytest.fixture(scope="module")
def r8_manifest():
    with open(os.path.join(GOLDEN_DIR, "manifest_r8.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("name", CASES)
def test_forward_r8_matches_reference_golden(name, r8_manifest, model):
    report_checks(name, model, golden_checks(model, r8_manifest[name], load_golden(name)))


@pytest.mark.parametrize("name", CASES)
def test_forward_r8_volume_free_raft_matches_reference_golden(name, r8_manifest, weights0, monkeypatch):
    """RAFT's lookups computed on the fly from the other frame's pooled half-precision features (no all-pairs volume; forced here,
    chosen by size otherwise) on the odd grids, where the pooled feature levels floor odd sizes (17 -> 8 -> 4 -> 2)."""
    monkeypatch.setenv("GIMMVFI_RAFT_CORR_DIRECT", "1")       # read when the engine is created
    m = GIMMVFI_R(seed=0).to(DEV).eval()
    m.load_state_dict(weights0, strict=True)
    report_checks(name + " volume-free RAFT", m, golden_checks(m, r8_manifest[name], load_golden(name)))
