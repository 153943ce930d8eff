"""Parameter inventory of GIMM-VFI-R: the 414-tensor ``state_dict`` layout the
drop-in module must accept unchanged (reference: gimmvfi_r.py:37-111,
raft/extractor.py:122-171, raft/update.py:94-154, modules/fi_components.py,
modules/hyponet.py:148-186; SURVEY.md §8(b) "Checkpoint layout").

``param_spec_r()`` returns ``[(key, shape, dtype_name)]`` in the reference's
state_dict order.  tests/test_arch.py checks it against
tests/golden/state_dict_spec_r.json, which was dumped from the reference.
"""
from typing import List, Tuple

Spec = List[Tuple[str, tuple, str]]


def _conv(out: Spec, name: str, cout: int, cin: int, kh: int, kw: int = None):
    kw = kh if kw is None else kw
    out.append((name + ".weight", (cout, cin, kh, kw), "float32"))
    out.append((name + ".bias", (cout,), "float32"))


def _bn(out: Spec, name: str, c: int):
    out.append((name + ".weight", (c,), "float32"))
    out.append((name + ".bias", (c,), "float32"))
    out.append((name + ".running_mean", (c,), "float32"))
    out.append((name + ".running_var", (c,), "float32"))
    out.append((name + ".num_batches_tracked", (), "int64"))


def _prelu(out: Spec, name: str, c: int):
    out.append((name + ".weight", (c,), "float32"))


def _convrelu(out: Spec, name: str, cout: int, cin: int, k: int):
    _conv(out, name + ".0", cout, cin, k)
    _prelu(out, name + ".1", cout)


def _raft_encoder(out: Spec, p: str, batchnorm: bool):
    """raft/extractor.py:122-171 — InstanceNorm2d has no parameters/buffers."""
    if batchnorm:
        _bn(out, p + ".norm1", 64)
    _conv(out, p + ".conv1", 64, 3, 7)
    cin = 64
    for li, dim in ((1, 64), (2, 96), (3, 128)):
        for bi in (0, 1):
            q = "%s.layer%d.%d" % (p, li, bi)
            down = bi == 0 and li > 1
            _conv(out, q + ".conv1", dim, cin if bi == 0 else dim, 3)
            _conv(out, q + ".conv2", dim, dim, 3)
            if batchnorm:
                _bn(out, q + ".norm1", dim)
                _bn(out, q + ".norm2", dim)
                if down:
                    _bn(out, q + ".norm3", dim)
            if down:
                _conv(out, q + ".downsample.0", dim, cin, 1)
                if batchnorm:
                    _bn(out, q + ".downsample.1", dim)  # same module object as norm3
        cin = dim
    _conv(out, p + ".conv2", 256, 128, 1)


def _resblock(out: Spec, p: str, c: int, side: int):
    _convrelu(out, p + ".conv1", c, c, 3)
    _convrelu(out, p + ".conv2", side, side, 3)
    _convrelu(out, p + ".conv3", c, c, 3)
    _convrelu(out, p + ".conv4", side, side, 3)
    _conv(out, p + ".conv5", c, c, 3)
    _prelu(out, p + ".prelu", c)


def _amt_update(out: Spec, p: str):
    """fi_components.py:157-205 with the ctor args of gimmvfi_r.py:113-124."""
    _conv(out, p + ".convc1", 256, 648, 1)
    _conv(out, p + ".convc2", 192, 256, 3)
    _conv(out, p + ".convf1", 128, 4, 7)
    _conv(out, p + ".convf2", 64, 128, 3)
    _conv(out, p + ".conv", 188, 256, 3)
    _conv(out, p + ".gru.0", 192, 320, 3)
    _conv(out, p + ".gru.2", 192, 192, 3)
    _conv(out, p + ".feat_head.0", 192, 192, 3)
    _conv(out, p + ".feat_head.2", 128, 192, 3)
    _conv(out, p + ".flow_head.0", 192, 192, 3)
    _conv(out, p + ".flow_head.2", 4, 192, 3)


def param_spec_r() -> Spec:
    s: Spec = []
    s.append(("g_filter", (1, 1, 1, 3, 3), "float32"))
    s.append(("alpha_v", (1,), "float32"))
    s.append(("alpha_fe", (1,), "float32"))
    _raft_encoder(s, "flow_estimator.fnet", False)
    _raft_encoder(s, "flow_estimator.cnet", True)
    u = "flow_estimator.update_block"
    _conv(s, u + ".encoder.convc1", 256, 324, 1)
    _conv(s, u + ".encoder.convc2", 192, 256, 3)
    _conv(s, u + ".encoder.convf1", 128, 2, 7)
    _conv(s, u + ".encoder.convf2", 64, 128, 3)
    _conv(s, u + ".encoder.conv", 126, 256, 3)
    for sfx, kh, kw in (("1", 1, 5), ("2", 5, 1)):
        for gate in "zrq":
            _conv(s, "%s.gru.conv%s%s" % (u, gate, sfx), 128, 384, kh, kw)
    _conv(s, u + ".flow_head.conv1", 256, 128, 3)
    _conv(s, u + ".flow_head.conv2", 2, 256, 3)
    _conv(s, u + ".mask.0", 256, 128, 3)
    _conv(s, u + ".mask.2", 576, 256, 1)
    _conv(s, "amt_last_cproj", 256, 128, 1)
    _conv(s, "amt_second_last_cproj", 128, 96, 1)
    _conv(s, "amt_fproj", 256, 256, 1)
    # NewInitDecoder(256, 64)  fi_components.py:229-253
    p = "amt_init_decoder"
    _convrelu(s, p + ".upsample.1", 64, 64, 5)
    for i in (2, 3, 4):
        _convrelu(s, "%s.upsample.%d" % (p, i), 64, 64, 3)
    _convrelu(s, p + ".upsample.5", 128, 64, 3)
    _conv(s, p + ".upsample.6", 128, 128, 1)
    _bn(s, p + ".upsample.7", 128)
    _convrelu(s, p + ".convblock.0", 128, 272, 1)
    for i in (1, 2, 3):
        _resblock(s, "%s.convblock.%d" % (p, i), 128, 64)
    _conv(s, p + ".convblock.4", 133, 128, 3)
    # NewMultiFlowDecoder(128, 64)  fi_components.py:279-305
    p = "amt_final_decoder"
    _convrelu(s, p + ".upsample.2", 32, 8, 5)
    for i in (3, 4, 5):
        _convrelu(s, "%s.upsample.%d" % (p, i), 32, 32, 3)
    _convrelu(s, p + ".upsample.6", 64, 32, 3)
    _conv(s, p + ".upsample.7", 64, 64, 1)
    _bn(s, p + ".upsample.8", 64)
    _convrelu(s, p + ".convblock.0", 256, 273, 3)
    for i in (1, 2, 3):
        _resblock(s, "%s.convblock.%d" % (p, i), 256, 64)
    _conv(s, p + ".convblock.4", 24, 256, 3)
    _amt_update(s, "amt_update4_low")
    _amt_update(s, "amt_update4_high")
    _conv(s, "amt_comb_block.0", 18, 9, 7)
    _prelu(s, "amt_comb_block.1", 18)
    _conv(s, "amt_comb_block.2", 3, 18, 7)
    # cnn_encoder gimmvfi_r.py:86-97
    _conv(s, "cnn_encoder.0", 16, 2, 3)
    _conv(s, "cnn_encoder.1", 32, 16, 3)
    for i in (3, 4, 5):
        _conv(s, "cnn_encoder.%d.layers.0" % i, 32, 32, 3)
        _conv(s, "cnn_encoder.%d.layers.2" % i, 32, 32, 3)
    _conv(s, "cnn_encoder.7", 16, 32, 3)
    # res_conv gimmvfi_r.py:100-109
    _conv(s, "res_conv.0", 32, 64, 3)
    _conv(s, "res_conv.1", 64, 32, 3)
    _conv(s, "res_conv.3.layers.0", 64, 64, 3)
    _conv(s, "res_conv.3.layers.2", 64, 64, 3)
    _conv(s, "res_conv.5", 32, 64, 3)
    # HypoNet hyponet.py:148-169: (32+3+1,128), (129,128)x3, (129,2)
    s.append(("hyponet.params_dict.linear_wb0", (36, 128), "float32"))
    for i in (1, 2, 3):
        s.append(("hyponet.params_dict.linear_wb%d" % i, (129, 128), "float32"))
    s.append(("hyponet.params_dict.linear_wb4", (129, 2), "float32"))
    return s


R_ONLY_PREFIXES = ("flow_estimator.", "amt_last_cproj.", "amt_second_last_cproj.", "amt_fproj.")
ESTIMATOR_PREFIX = "flow_estimator."


def strip_prefix(spec: Spec) -> Spec:
    """the `flow_estimator.*` entries of a GIMM-VFI spec in registration order, prefix stripped: the spec of the estimator module
    alone (RAFT for param_spec_r, FlowFormer for param_spec_f)"""
    return [(k[len(ESTIMATOR_PREFIX):], s, dt) for k, s, dt in spec if k.startswith(ESTIMATOR_PREFIX)]


def param_spec_f() -> Spec:
    """GIMM-VFI-F (gimmvfi_f.py:27-111): 639 tensors = FlowFormer (`flow_estimator.*`: Twins-SVT-L stages 1-2 x2, cost-perceiver
    encoder, GMA memory decoder — flowformer/core/**) + the same decoder / GIMM parameter tree as GIMM-VFI-R without its three feature
    projections.  The FlowFormer part (410 keys, the layout of its published `flowformer_sintel.pth` checkpoint) is kept as a
    schema table (specs/state_dict_spec_f.json, dumped from the reference module; tests/test_arch.py compares it with the dump
    under tests/golden/); the rest is generated exactly like param_spec_r."""
    import json
    import os

    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "specs", "state_dict_spec_f.json")) as f:
        table = json.load(f)
    spec = [(k, tuple(shape), dt) for k, shape, dt in table]
    shared = {k: (shape, dt) for k, shape, dt in param_spec_r() if not k.startswith(R_ONLY_PREFIXES)}
    for k, shape, dt in spec:   # the synthesis half must be the R layout, key for key
        if not k.startswith("flow_estimator."):
            assert k in shared and tuple(shared[k][0]) == tuple(shape) and shared[k][1] == dt, k
    assert sum(1 for k, _, _ in spec if not k.startswith("flow_estimator.")) == len(shared)
    return spec
