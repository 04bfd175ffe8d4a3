"""CPU: the engine's host-side sequencing against a recording stand-in for the C ABI (no kernels
run): which entry points a train step calls in each mode, that the device pointer tables are
complete before a step (a CUDA-graph capture cannot contain their host-to-device copy), and the
bookkeeping of the in-place weight-gradient accumulation."""
import pytest
import torch

import oracle.ae_oracle as orc


class RecordingLib:
    """Every avc_* call succeeds and is recorded; size queries answer plausibly."""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def f(*a):
            self.calls.append(name)
            if name in ("avc_tc_packed_floats", "avc_wgrad_tc_scratch_floats", "avc_conv_wgrad_scratch_floats"):
                return 64
            if name == "avc_wgrad_acc_floats":
                return a[2] * a[1] * (((a[0] + 127) // 128) * 128)
            return 0
        return f


@pytest.fixture()
def rig(monkeypatch):
    from adaptive_voice_conversion_b200 import engine as E
    cfg = orc.default_config(80)
    e = object.__new__(E.Engine)      # the real constructor insists on a CUDA device
    e.cfg, e.dev, e.lib, e.packed, e.debug = cfg, torch.device("cpu"), RecordingLib(), {}, None
    e.precision, e.tc_status, e._packed_key = "tf32", torch.zeros(1, dtype=torch.int32), None
    e._init_options()
    e.fused_dense, e.wgrad_acc, e.fold_fused = True, False, False
    monkeypatch.setattr(E.Engine, "stream", property(lambda self: 0))
    monkeypatch.setattr(E.Engine, "zeros", lambda self, *shape: torch.zeros(shape))
    P = orc.init_state(cfg, seed=0)
    G = {k: torch.zeros_like(v) for k, v in P.items()}
    e.pack_weights(P, need_dgrad=True)
    return e, P, G


def full_step(e, P, G):
    x = torch.randn(4, 80, 128)
    emb, cs = e.speaker_fwd(P, x, True)
    mu4, ls4, ce = e.content_fwd(P, x, True)
    eps = torch.randn(4, 128, 16)
    mu, ls, z4 = e.reparam_fwd(mu4, ls4, eps)
    dec4, cd = e.decoder_fwd(P, z4, emb, True)
    from adaptive_voice_conversion_b200.engine import A4
    dz4, demb = e.decoder_bwd(P, G, cd, A4.empty(dec4.B, dec4.C, dec4.T, e.dev))
    dmu4, dls4 = e.reparam_bwd(dz4, ls4, eps, torch.zeros_like(mu), torch.zeros_like(ls))
    e.content_bwd(P, G, ce, dmu4, dls4)
    e.speaker_bwd(P, G, cs, demb)
    e.flush_wgrad()
    return emb, demb


def test_fused_dense_replaces_the_per_layer_linears(rig):
    e, P, G = rig
    e.lib.calls.clear()
    emb, demb = full_step(e, P, G)
    c = e.lib.calls
    assert emb.shape == (4, 128) and demb.shape == (4, 128)
    assert c.count("avc_dense_stack_fwd") == 1 and c.count("avc_dense_stack_bwd") == 1
    assert c.count("avc_linear_batch_fwd") == 1 and c.count("avc_linear_batch_dx") == 1 and c.count("avc_linear_batch_dw") == 2
    assert not any(n in ("avc_linear_fwd", "avc_linear_bwd") for n in c)
    e.fused_dense = False
    e.lib.calls.clear()
    full_step(e, P, G)
    assert e.lib.calls.count("avc_linear_fwd") == 25 and e.lib.calls.count("avc_linear_bwd") == 25
    assert "avc_dense_stack_fwd" not in e.lib.calls


def test_pointer_tables_are_complete_before_a_step(rig):
    e, P, G = rig
    e.prepare_tables(P, G)
    before = {k: id(v[1]) for k, v in e._ptr_tables.items()}
    assert len(before) == 6      # params + grads of the dense stack and of the affine layers, bank bias gradients of both encoders
    full_step(e, P, G)
    assert {k: id(v[1]) for k, v in e._ptr_tables.items()} == before      # nothing was (re)built mid-step
    # a moved parameter invalidates its table
    P["decoder.conv_affine_layers.3.bias"] = P["decoder.conv_affine_layers.3.bias"].clone()
    e.prepare_tables(P, G)
    after = {k: id(v[1]) for k, v in e._ptr_tables.items()}
    changed = [k for k in before if before[k] != after[k]]
    assert changed == [("params", "decoder.conv_affine_layers.0")]


def test_wgrad_accumulation_bookkeeping(rig):
    e, P, G = rig
    e.wgrad_acc = True
    e.prepare_wgrad_acc(P, G)
    acc = e._wg_acc
    assert acc is not None and acc["n"] == 58 and not acc["dirty"]
    # regions are disjoint and cover the arena
    offs = sorted(acc["offs"].values())
    assert offs[0] == 0 and len(set(offs)) == len(offs) and acc["arena"].numel() > offs[-1]
    e.lib.calls.clear()
    full_step(e, P, G)
    c = e.lib.calls
    assert c.count("avc_conv_wgrad_tc_acc") == 58 and c.count("avc_conv_wgrad_tc") == 0 and c.count("avc_wgrad_acc_flush") == 1
    assert not acc["dirty"]
    # gradients in OTHER buffers (the autograd path allocates its own) must not use the registered arena
    G2 = {k: torch.zeros_like(v) for k, v in P.items()}
    e.lib.calls.clear()
    full_step(e, P, G2)
    assert e.lib.calls.count("avc_conv_wgrad_tc_acc") == 0 and e.lib.calls.count("avc_conv_wgrad_tc") == 58
    assert "avc_wgrad_acc_flush" not in e.lib.calls
    # switched off: registration is dropped
    e.wgrad_acc = False
    e.prepare_wgrad_acc(P, G)
    assert e._wg_acc is None


def test_decoder_accumulators_can_be_flushed_early(rig):
    """flush_wgrad(decoder_only=True) covers exactly the decoder's rows (the tail of the item table), the closing
    flush the rest; nothing is flushed twice and the flags reset for the next step (trainer.py: the decoder's weight
    gradients are folded on their own stream while the encoders' backward runs)."""
    e, P, G = rig
    e.wgrad_acc = True
    e.prepare_wgrad_acc(P, G)
    acc = e._wg_acc
    n_dec = sum(1 for n in e.conv_names() if n.startswith("decoder."))
    assert acc["n_dec"] == n_dec == 14
    seen = []
    real = e.lib.__getattr__("avc_wgrad_acc_flush")

    def flush(items, n, max_units, stream):
        seen.append((items - acc["items"].data_ptr(), n))
        return real(items, n, max_units, stream)
    e.lib.__dict__["avc_wgrad_acc_flush"] = flush
    from adaptive_voice_conversion_b200.engine import A4
    for _ in range(2):                                   # two steps: the flags must reset
        seen.clear()
        x = torch.randn(4, 80, 128)
        emb, cs = e.speaker_fwd(P, x, True)
        mu4, ls4, ce = e.content_fwd(P, x, True)
        eps = torch.randn(4, 128, 16)
        mu, ls, z4 = e.reparam_fwd(mu4, ls4, eps)
        dec4, cd = e.decoder_fwd(P, z4, emb, True, affine=e.decoder_affine_fwd(P, emb, True))
        dz4, demb = e.decoder_bwd(P, G, cd, A4.empty(dec4.B, dec4.C, dec4.T, e.dev))
        e.flush_wgrad(decoder_only=True)
        e.flush_wgrad(decoder_only=True)                 # idempotent
        dmu4, dls4 = e.reparam_bwd(dz4, ls4, eps, torch.zeros_like(mu), torch.zeros_like(ls))
        e.content_bwd(P, G, ce, dmu4, dls4)
        e.speaker_bwd(P, G, cs, demb)
        e.join_wgrad()
        e.flush_wgrad()
        item = 32                                        # sizeof(avc_wgrad_acc_item)
        assert seen == [((58 - n_dec) * item, n_dec), (0, 58 - n_dec)]
        assert not acc["dirty"] and not acc["dec_done"]
    # without the early call the closing flush takes every row
    seen.clear()
    full_step(e, P, G)
    assert seen == [(0, 58)]


def test_fused_fold_drops_the_fold_launches(rig):
    e, P, G = rig
    e.lib.calls.clear()
    full_step(e, P, G)
    n_fold, n_conv = e.lib.calls.count("avc_fold_add_fwd"), e.lib.calls.count("avc_conv_block_tc")
    assert n_fold > 30
    e.fold_fused = True
    e.lib.calls.clear()
    full_step(e, P, G)
    # left: the 6 stride-2 data gradients (even/odd tap convs) and the one plain tensor add of content_bwd
    assert e.lib.calls.count("avc_fold_add_fwd") == 7 and e.lib.calls.count("avc_conv_block_tc") == n_conv
    assert n_fold - 7 == 30
