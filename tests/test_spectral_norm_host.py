"""CPU: the decoder's spectral norm (Decoder.sn) -- the reference's checkpoint layout, its seeded initialisation, its
optimizer parameter order, and the float64 restatement of the power iteration and its adjoint that the GPU tests
measure the kernels against."""
import ctypes
import os
import subprocess
import tempfile

import pytest
import torch

from _sn_ref import adjoint64, power_iteration64, sn_config, state_checksum
from conftest import GOLDEN, ROOT
from oracle.make_golden import load_fixture

REF = os.environ.get("AVC_REFERENCE_DIR", "")


def fixture(name="train_sn_c80_b4.pt"):
    return load_fixture(os.path.join(GOLDEN, name))


def build_ae(seed=0, c_in=80):
    from adaptive_voice_conversion_b200.model import AE
    torch.manual_seed(seed)
    return AE(sn_config(c_in))


def test_state_dict_layout_matches_the_reference():
    """218 entries: bias, weight_orig, weight_u, weight_v for each of the 26 wrapped decoder layers, in the
    reference's order, with the spectral_norm version metadata."""
    fx = fixture()
    sd = build_ae().state_dict()
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == fx["state_keys"]
    assert len(sd) == 218
    meta = {k: dict(v) for k, v in sd._metadata.items() if "spectral_norm" in v}
    assert meta == fx["state_metadata"] and len(meta) == 26


def test_initialisation_is_the_references_seed_for_seed():
    """torch.manual_seed(0); AE(cfg) draws every weight and then u, v in the reference's module order."""
    for name in ("train_sn_c80_b4.pt", "infer_sn_c80.pt"):
        fx = fixture(name)
        ae = build_ae(fx["init_seed"])
        assert torch.equal(state_checksum(ae.state_dict()), fx["state_checksum"])
        mods = dict(ae.named_modules())
        for n, rec in fx["sn_init"].items():
            assert torch.equal(mods[n].weight_u, rec["u"]) and torch.equal(mods[n].weight_v, rec["v"]), n


def test_parameter_order_is_the_references():
    """ae.parameters() -- what a .opt file's integer keys index -- lists bias before weight_orig in a wrapped layer."""
    fx = fixture()
    ae = build_ae()
    assert [n for n, _ in ae.named_parameters()] == fx["param_names"]
    assert fx["param_names"].index("decoder.in_conv_layer.bias") + 1 == fx["param_names"].index("decoder.in_conv_layer.weight_orig")


def test_sn_false_layout_is_unchanged():
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200.model import AE
    cfg = orc.default_config(80)
    sd = AE(cfg).state_dict()
    assert list(sd) == list(orc.init_state(cfg, seed=0)) and len(sd) == 166


@pytest.mark.skipif(not REF or not os.path.isdir(REF), reason="set AVC_REFERENCE_DIR to a checkout of the original project")
def test_against_the_live_reference():
    """Strict load_state_dict in both directions, the same state_dict seed for seed, the same parameter order."""
    from oracle.make_golden import import_reference
    ref_model = import_reference()
    for seed in (0, 3):
        torch.manual_seed(seed)
        ref = ref_model.AE(sn_config(80))
        ours = build_ae(seed)
        rsd, osd = ref.state_dict(), ours.state_dict()
        assert list(rsd) == list(osd) and all(torch.equal(rsd[k], osd[k]) for k in rsd)
        sn_meta = lambda sd: {k: dict(v) for k, v in sd._metadata.items() if "spectral_norm" in v}   # noqa: E731
        assert sn_meta(rsd) == sn_meta(osd) and len(sn_meta(osd)) == 26
        assert [n for n, _ in ref.named_parameters()] == [n for n, _ in ours.named_parameters()]
        ours.load_state_dict(rsd, strict=True)
        ref.load_state_dict(osd, strict=True)


@pytest.mark.parametrize("kind", ["conv_k5", "conv_k1", "linear"])
@pytest.mark.parametrize("training", [True, False])
def test_float64_restatement_equals_torch_autograd(kind, training):
    """The restatement (power iteration, sigma, W / sigma, and the gradient with u, v held constant) equals torch's
    spectral_norm hook and autograd through it, both in double."""
    torch.manual_seed(11)
    m = {"conv_k5": lambda: torch.nn.Conv1d(24, 40, 5), "conv_k1": lambda: torch.nn.Conv1d(24, 40, 1),
         "linear": lambda: torch.nn.Linear(24, 40)}[kind]().double()
    m = torch.nn.utils.spectral_norm(m)
    for _ in range(2):                      # u, v away from their random start
        m.train()
        m(torch.randn(2, 24, 9, dtype=torch.float64) if kind != "linear" else torch.randn(2, 24, dtype=torch.float64))
    W, u0, v0 = m.weight_orig.detach().clone(), m.weight_u.clone(), m.weight_v.clone()
    m.train(training)
    m(torch.randn(2, 24, 9, dtype=torch.float64) if kind != "linear" else torch.randn(2, 24, dtype=torch.float64))
    R = torch.randn(W.shape, dtype=torch.float64)
    (m.weight * R).sum().backward()
    u, v, sigma, W_bar = power_iteration64(W, u0, v0, iterate=training)
    assert float((u - m.weight_u).abs().max()) < 1e-12 and float((v - m.weight_v).abs().max()) < 1e-12
    assert float((W_bar - m.weight.detach()).abs().max()) < 1e-12
    g = adjoint64(R, W_bar, u, v, sigma)
    assert float((g - m.weight_orig.grad).abs().max()) < 1e-12 * float(g.abs().max())


def test_sn_item_layout_matches_the_header():
    from adaptive_voice_conversion_b200 import _lib as L
    prog = '#include <stdio.h>\n#include "avc_b200.h"\nint main(){printf("%zu %d %d %d\\n", sizeof(avc_sn_item), AVC_SN_MAX_ITEMS, AVC_SN_MAX_H, AVC_SN_MAX_W);return 0;}\n'
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "s.c")
        open(c, "w").write(prog)
        exe = os.path.join(td, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        vals = [int(v) for v in subprocess.check_output([exe]).split()]
    assert vals == [ctypes.sizeof(L.SnItem), L.SN_MAX_ITEMS, L.SN_MAX_H, L.SN_MAX_W]
    lib = L.load()
    assert lib.avc_spectral_norm_scratch_floats(256, 640) == 16 * 640 + 256 + 16
    # argument checks need no device: they return before any launch
    assert lib.avc_spectral_norm(None, 1, 8, 8, L.SN_ITERATE, None, None) == L.ERR_INVALID
    assert lib.avc_spectral_norm(1, 1, L.SN_MAX_H + 1, 8, L.SN_ITERATE, 1, None) == L.ERR_UNSUPPORTED
    assert lib.avc_spectral_norm(1, L.SN_MAX_ITEMS + 1, 8, 8, L.SN_FIXED, 1, None) == L.ERR_UNSUPPORTED
    assert lib.avc_spectral_norm(1, 1, 8, 8, 7, 1, None) == L.ERR_INVALID
    assert lib.avc_spectral_norm_bwd(1, 1, 8, L.SN_MAX_W + 1, 1, None) == L.ERR_UNSUPPORTED
