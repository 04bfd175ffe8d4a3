"""GPU: every layer of a training step and of inference against tests/_layer_ref.py's float64 restatement of that
layer, on the engine's own fp32 inputs to it.

The end-to-end parity tests (test_gpu_model.py, test_gpu_tf32_accuracy.py) have to be loose, because a ReLU that flips
anywhere moves every later value (DESIGN.md section 6).  Here each layer is checked locally: hooks on Engine.conv,
Engine.conv_bwd, the engine's debug callback and a few stack entry points clone what each layer read and wrote (on the
stream it ran on, right behind its launch); the float64 chain of _layer_ref.py then runs with a tap that compares its
value at each boundary with the engine's and continues with the engine's.  The reference's inputs are semantic: a block's
residual is the previous layer's captured output, a decoder layer's AdaIN row is the float64 affine of the captured
speaker embedding, a layer's upstream gradient is built from the downstream layers' captured gradients.  So a wrong
pointer, row, residual mode or flag shows up as an error at the layer that has it.

- A launch that ran on the tensor cores (avc_conv_block_tc, avc_conv_wgrad_tc, avc_conv_wgrad_tc_acc; a proxy of the
  engine's library records which layer made each launch) is compared with a reference whose conv operands are rounded to
  TF32 as the kernel rounds them.  An FFMA launch inside a TF32 step (the weight and data gradients of layers longer
  than the tensor-core kernels take) is compared with the captured operands as they are: dc is already TF32-rounded
  where the engine rounded it (F_ROUND_OUT), the rest is raw fp32.
- Every buffer the engine marks TF32-exact (A4.tf32: a consumer then skips its own rounding) must be TF32-exact.
- ReLU ambiguity: an element whose float64 pre-activation is within TAU of its row's largest is ambiguous; the engine
  may take either branch there (per element forward, per row in the backward, at most 4 per row).
- Errors are measured against the magnitude of the terms (Σ|x||dc| for weight gradients) or of the reference tensor
  (outputs, raw-output gradients, AdaIN rows), after half a TF32 ulp of each element where the engine rounds it.
- The instrumented step gives the same bits (gradients, losses, updated parameters) as an uninstrumented one, every
  parameter is checked by exactly one layer or unit, and every conv-family launch belongs to a checked layer.
"""
import contextlib
import io
import itertools
import types
from collections import defaultdict

import pytest
import torch

import _layer_ref as LR
import oracle.ae_oracle as orc
from _sn_ref import sn_config

pytestmark = pytest.mark.gpu

TAU = 1e-5
MAX_AMB_PER_ROW = 4
# about 3x the worst measured on 1x H100 80GB HBM3 (700 W power limit), over every case of this file:
#   fp32: fwd 5.5e-6 (inference, 17 frames), dc 1.3e-6, dx 1.4e-6, dw 6.7e-7, grad 4.2e-7, misc 1.5e-6
#   tf32: fwd 1.1e-5 (inference, 1000 frames), dc 1.8e-6, dx 4.0e-6, dw 2.5e-6, grad 3.2e-7, misc 5.5e-6
# The weight-gradient error grows with the length of its reduction over batch and time: the TF32 worst, 2.5e-6, is the
# speaker encoder's in_conv at B = 37 (4736 terms per weight); at B = 8 no layer exceeds 8.0e-7.
# ambiguous ReLU elements (|pre| < TAU of the row's largest) per training step: 79-97 at B = 8, 437 at B = 37;
# per inference call (3 pairs): 2-221
# Segments of other lengths (same card), worst of fwd / dc / dx / dw / grad / misc:
#   T = 64:  fp32 2.3e-6 / 1.9e-6 / 1.2e-6 / 5.4e-7 / 3.6e-7 / 1.5e-6   tf32 3.4e-6 / 1.2e-6 / 3.2e-6 / 7.0e-7 / 5.0e-7 / 3.4e-6
#   T = 200: fp32 2.7e-6 / 1.0e-6 / 1.7e-6 / 1.0e-6 / 3.1e-7 / 1.4e-6   tf32 2.3e-6 / 8.2e-7 / 3.9e-6 / 9.9e-7 / 4.2e-7 / 3.6e-6
#   T = 256: fp32 2.5e-6 / 1.3e-6 / 1.5e-6 / 5.9e-7 / 4.2e-7 / 9.4e-7   tf32 2.6e-6 / 1.4e-6 / 4.0e-6 / 8.2e-7 / 3.5e-7 / 4.8e-6
#            tf32 c512 6.1e-6 / 2.0e-6 / 4.0e-6 / 7.3e-7 / 2.7e-7 / 4.1e-6, sn 2.6e-6 / 1.6e-6 / 3.4e-6 / 7.3e-7 / 3.1e-7 / 3.6e-6
#   T = 512 (B = 4): fp32 2.1e-6 / 1.1e-6 / 1.4e-6 / 6.7e-7 / 5.1e-7 / 1.1e-6   tf32 2.7e-6 / 1.2e-6 / 3.8e-6 / 8.1e-7 / 7.4e-7 / 4.2e-6
# (dw at B·T = 1600-2048 terms per weight stays below 1.0e-6, in the FFMA weight gradient the TF32 step takes there too);
# ambiguous elements per step 42-45 at T = 64, 151-207 at 200 and 256, 208-228 at 512.
TOL = {"fp32": dict(fwd=2e-5, dc=5e-6, dx=5e-6, dw=2e-6, grad=1.5e-6, misc=5e-6),
       "tf32": dict(fwd=3.5e-5, dc=6e-6, dx=1.2e-5, dw=7.5e-6, grad=1.5e-6, misc=2e-5)}
TC_FWD = ("avc_conv_block_tc",)
TC_WGRAD = ("avc_conv_wgrad_tc", "avc_conv_wgrad_tc_acc")
CONV_FAMILY = ("avc_conv_block_tc", "avc_conv_block_fwd", "avc_norm_bwd", "avc_norm_apply_fwd", "avc_conv_wgrad",
               "avc_conv_wgrad_tc", "avc_conv_wgrad_tc_acc", "avc_bias_grad")


def planar(a):
    """A4 (possibly a channel range of a wider buffer) -> a [B][C][T] clone, on the current stream."""
    ctot = a.t.shape[1] * 4
    c0 = (a.ptr - a.t.data_ptr()) // (a.T * 16) * 4
    return a.t.permute(0, 1, 3, 2).reshape(a.B, ctot, a.T)[:, c0:c0 + a.C].clone()


class RecordingLib:
    """The engine's library, with every avc_* call recorded together with the layer that made it."""

    def __init__(self, lib, cap):
        self._lib, self._cap = lib, cap

    def __getattr__(self, n):
        f = getattr(self._lib, n)
        if not n.startswith("avc_"):
            return f

        def call(*a):
            self._cap.launches.append((n, self._cap.cur))
            return f(*a)
        return call


class Capture:
    def __init__(self):
        self.fwd, self.dc, self.dx, self.launches = {}, {}, {}, []
        self.cur, self.emb, self.demb, self.dconds, self.sn, self.wbar = None, None, None, None, {}, {}

    def tagged(self, tag, fn):
        prev, self.cur = self.cur, tag
        try:
            return fn()
        finally:
            self.cur = prev

    def tc(self, name, op):
        if op == "fwd":
            return any(n in TC_FWD and t == (name, "fwd") for n, t in self.launches)
        if op == "dgrad":
            return any(n in TC_FWD and t == (name, "bwd") for n, t in self.launches)
        return any(n in TC_WGRAD and t == (name, "wgrad") for n, t in self.launches)


def install(monkeypatch, eng, cap):
    from adaptive_voice_conversion_b200 import engine as E
    Eng = E.Engine
    conv0, bwd0, wg0 = Eng.conv, Eng.conv_bwd, Eng._wgrad_launch
    sfwd0, sbwd0, aff0, sn0, snb0 = Eng.speaker_fwd, Eng.speaker_bwd, Eng._decoder_affine_bwd, Eng.spectral_norm, Eng.spectral_norm_bwd

    def conv(self, P, name, xin, **kw):
        out, rec = cap.tagged((name, "fwd"), lambda: conv0(self, P, name, xin, **kw))
        cond = kw.get("cond")
        # (a bank conv rounds its output into its channel range of the concat: that view carries no tf32 flag)
        rounded = out.tf32 or (kw.get("round_out", False) and self.precision == "tf32" and not self.fwd_fp32)
        # a padded batch: the valid frames of xin, and of out before a pixel shuffle doubles them
        lens = kw.get("lens")
        lo = None if lens is None else lens.down(kw.get("stride", 1))
        cap.fwd[name] = dict(x=planar(xin), x_tf32=xin.tf32, out=planar(out), out_tf32=out.tf32, rounded=rounded,
                             cond=None if cond is None else cond.clone(), shuffle=kw.get("shuffle", False),
                             lens=None if lens is None else (lens.t.clone(), lens.div, lens.mul),
                             lens_out=None if lo is None else (lo.t.clone(), lo.div, lo.mul))
        return out, rec

    def conv_bwd(self, P, G, rec, dy, **kw):
        name = rec["name"]
        if not (rec["norm"] or rec["relu"]) and kw.get("dc_pre") is None:
            cap.dc[name] = (planar(dy), dy.tf32)
        r = cap.tagged((name, "bwd"), lambda: bwd0(self, P, G, rec, dy, **kw))
        if r is not None:
            cap.dx[name] = planar(r)
        return r

    def wgrad_launch(self, wd, name):
        return cap.tagged((name, "wgrad"), lambda: wg0(self, wd, name))

    def speaker_fwd(self, P, x, train, lens=None, groups=None):
        emb, ctx = sfwd0(self, P, x, train, lens, groups)
        cap.emb = emb.clone()
        return emb, ctx

    def speaker_bwd(self, P, G, ctx, demb):
        cap.demb = demb.clone()
        return sbwd0(self, P, G, ctx, demb)

    def affine_bwd(self, P, G, ctx, dconds):
        cap.dconds = dconds.clone()
        return aff0(self, P, G, ctx, dconds)

    def sn_fwd(self, P, iterate):
        sn0(self, P, iterate)
        for n in self.sn_names():
            cap.wbar[n] = (P[n + ".weight"].clone(), iterate)

    def sn_bwd(self, P, G):
        for n in self.sn_names():
            cap.sn[n] = (P[n + ".weight"].clone(), G[n + ".weight"].clone())
        return snb0(self, P, G)

    def debug(name, stage, obj):
        if stage == "dc":
            cap.dc[name] = (planar(obj), obj.tf32)

    for attr, f in (("conv", conv), ("conv_bwd", conv_bwd), ("_wgrad_launch", wgrad_launch), ("speaker_fwd", speaker_fwd),
                    ("speaker_bwd", speaker_bwd), ("_decoder_affine_bwd", affine_bwd), ("spectral_norm", sn_fwd),
                    ("spectral_norm_bwd", sn_bwd)):
        monkeypatch.setattr(Eng, attr, f)
    monkeypatch.setattr(eng, "debug", debug)
    monkeypatch.setattr(eng, "lib", RecordingLib(eng.lib, cap))


def tf32_exact(t):
    return bool(((t.contiguous().view(torch.int32) & 0x1FFF) == 0).all())


class Checker:
    """The tap: compares the reference at each boundary with the engine's captured value, records the error (worst per
    kind and per layer) and returns the value the chain continues with."""

    def __init__(self, cap, G, cfg, tf32):
        self.cap, self.G, self.cfg, self.tf32 = cap, G, cfg, tf32
        self.worst = defaultdict(float)
        self.where = {}
        self.checked = defaultdict(int)
        self.amb = 0
        self.problems = []

    def err(self, kind, unit, e):
        e = float(e)
        w = self.worst.get(kind)
        # NaN counts as worse than anything, and stays the worst once recorded (a later e <= NaN is False too)
        if w is None or (w == w and not (e <= w)):
            self.worst[kind], self.where[kind] = e, unit

    def honest(self, what, t, flag):
        if flag and not tf32_exact(t):
            self.problems.append(f"{what} is marked TF32-exact but is not")

    def _ambiguous(self, name, pre):
        amb = pre.abs() < TAU * pre.abs().amax(dim=2, keepdim=True)
        n = amb.sum(dim=2)
        if int(n.max()) > MAX_AMB_PER_ROW:
            self.problems.append(f"{name}: {int(n.max())} ambiguous ReLU elements in one row")
        return amb

    @staticmethod
    def _rel(eng, ref, scale, allow=0.0):
        d = (eng.double() - ref.double()).abs() - allow
        return float(d.clamp_min(0).max()) / max(float(scale), 1e-30)

    def __call__(self, kind, name, ref, **info):
        cap = self.cap
        if kind == "out":
            f = cap.fwd[name]
            eng = f["out"].double()
            d = (eng - ref).abs()
            if info["relu"]:
                pre = info["pre"]
                amb = self._ambiguous(name, pre)
                if amb.any():
                    self.amb += int(amb.sum())
                    alt = info["redo"]((pre > 0) ^ amb)
                    d = torch.minimum(d, (eng - alt).abs())
            allow = LR.tf32_half_ulp(ref) if f["rounded"] else 0.0
            scale = max(float(ref.abs().max()), float(info["pre"].abs().max()))
            self.err("fwd", name, float((d - allow).clamp_min(0).max()) / scale)
            self.honest(name + " output", f["out"], f["out_tf32"])
            self.honest(name + " input", f["x"], f["x_tf32"])
            return eng
        if kind == "dc":
            s = info["spec"]
            if ".conv_bank." in name:
                enc = name.split(".")[0]
                cb = self.cfg["SpeakerEncoder" if enc == "speaker_encoder" else "ContentEncoder"]["c_bank"]
                i = int(name.split(".")[-1])
                eng, flag = cap.dx[enc + ".in_conv_layer"][:, i * cb:(i + 1) * cb], False
            else:
                eng, flag = cap.dc[name]
            eng = eng.double()
            dc, dcond = ref
            if s["relu"]:
                dc, dcond = self._resolve(name, s, eng, dc, dcond, info)
            allow = LR.tf32_half_ulp(dc) if flag else 0.0
            self.err("dc", name, self._rel(eng, dc, dc.abs().max(), allow))
            self.honest(name + " dc", cap.dc[name][0] if name in cap.dc else eng.float(), flag)
            return eng, dcond
        if kind == "dw":
            dw, db = ref
            s = info["spec"]
            gw, gb = self.G[name + ".weight"].double(), self.G[name + ".bias"].double()
            terms, _ = LR.conv_dw(info["x"].abs(), info["dc"].abs(), s["K"], s["stride"], info["tf32"])
            e = self._rel(gw, dw, terms.abs().max())
            if info["tf32"]:
                # an operand the engine did not round (the residual stream, a masked or loss gradient) reaches the
                # tensor cores truncated or rounded depending on the weight-gradient kernel's staging: either is accepted
                dw2, _ = LR.conv_dw(info["x"], info["dc"], s["K"], s["stride"], "rna")
                e = min(e, self._rel(gw, dw2, terms.abs().max()))
            self.err("dw", name, e)
            if s["norm"] and not s["shuffle"]:
                if gb.any():
                    self.problems.append(f"{name}: the bias gradient before an InstanceNorm is not exactly 0")
            else:
                # the engine sums its fp32 dc; a TF32-rounded copy of it may differ by half an ulp per element
                dcf = info["dc"]
                allow = LR.tf32_half_ulp(dcf).sum(dim=(0, 2)) if (name in cap.dc and cap.dc[name][1]) else 0.0
                self.err("dw", name + ".bias", self._rel(gb, db, dcf.abs().sum(dim=(0, 2)).max(), allow))
            self.checked[name + ".weight"] += 1
            self.checked[name + ".bias"] += 1
            return ref
        if kind == "dx":
            if name in cap.dx:     # (where the engine materialised it: not when a fused norm backward skipped it)
                self.err("dx", name, self._rel(cap.dx[name], ref, ref.abs().max()))
            return ref
        if kind == "grad":
            self.err("grad", name, self._rel(self.G[name], ref, ref.abs().max()))
            self.checked[name] += 1
            return ref
        if kind == "x":
            eng = cap.fwd[name + ".conv_bank.0"]["x"]
            allow = LR.tf32_half_ulp(ref) if self.tf32 else 0.0
            self.err("misc", name + " x", self._rel(eng, ref, ref.abs().max(), allow))
            return eng.double()
        if kind == "emb":
            self.err("misc", "emb", self._rel(cap.emb, ref, ref.abs().max()))
            return cap.emb.double()
        if kind == "conds":
            for l in range(self.cfg["Decoder"]["n_conv_blocks"]):
                for j, nm in ((2 * l, f"decoder.first_conv_layers.{l}"), (2 * l + 1, f"decoder.second_conv_layers.{l}")):
                    self.err("misc", f"conds[{j}]", self._rel(cap.fwd[nm]["cond"], ref[:, j], ref[:, j].abs().max()))
            return ref
        if kind == "z":
            f = cap.fwd["decoder.in_conv_layer"]
            eng = f["x"]
            allow = LR.tf32_half_ulp(ref) if self.tf32 else 0.0     # (packed into A4 by a rounding pack_a4)
            self.err("misc", "z", self._rel(eng, ref, ref.abs().max(), allow))
            return eng.double()
        if kind in ("ddec", "dmu", "dls"):
            layer = {"ddec": "decoder.out_conv_layer", "dmu": "content_encoder.mean_layer", "dls": "content_encoder.std_layer"}[kind]
            eng, flag = cap.dc[layer]
            allow = LR.tf32_half_ulp(ref) if flag else 0.0
            self.err("misc", kind, self._rel(eng, ref, ref.abs().max(), allow))
            self.honest(kind, eng, flag)
            return eng.double()
        if kind == "dconds":
            eng = cap.dconds.permute(1, 0, 2).double()
            for j in range(ref.shape[0]):
                self.err("misc", f"dconds[{j}]", self._rel(eng[j], ref[j], ref[j].abs().max()))
            return eng
        if kind == "demb":
            self.err("misc", "demb", self._rel(cap.demb, ref, ref.abs().max()))
            return cap.demb.double()
        raise AssertionError(kind)

    def _resolve(self, name, s, eng, dc, dcond, info):
        """Per row with ambiguous ReLU elements: the reference under the branch combination closest to the engine."""
        pre = info["pre"]
        amb = self._ambiguous(name, pre)
        if not amb.any():
            return dc, dcond
        base = pre > 0
        dc, dcond = dc.clone(), None if dcond is None else dcond.clone()
        p = pre.shape[1]
        for b, c in amb.any(dim=2).nonzero().tolist():
            ts = amb[b, c].nonzero().flatten().tolist()[:MAX_AMB_PER_ROW]
            rows = [2 * c, 2 * c + 1] if s["shuffle"] else [c]
            best = None
            for bits in itertools.product((False, True), repeat=len(ts)):
                m = base.clone()
                for t, flip in zip(ts, bits):
                    m[b, c, t] ^= flip
                dcm, dcondm = info["redo"](m)
                e = float((eng[b, rows] - dcm[b, rows]).abs().max())
                if best is None or e < best[0]:
                    best = (e, dcm, dcondm)
            dc[b, rows] = best[1][b, rows]
            if dcond is not None:
                dcond[b, [c, p + c]] = best[2][b, [c, p + c]]
        return dc, dcond


# ------------------------------------------------------------------ the training step
def _solver(cfg, B, seed=0):
    from adaptive_voice_conversion_b200.solver import Solver
    cfg = dict(cfg, data_loader=dict(cfg["data_loader"], batch_size=B))
    args = types.SimpleNamespace(data_dir="synthetic", train_set="", train_index_file="", logdir="/tmp/avc_log", load_model=False,
                                 load_opt=False, store_model_path=None, load_model_path=None, summary_steps=10 ** 9, save_steps=10 ** 9,
                                 tag="t", iters=0)
    torch.manual_seed(seed)
    with contextlib.redirect_stdout(io.StringIO()):
        s = Solver(cfg, args)
    if not cfg["Decoder"].get("sn", False):
        s.model.load_state_dict(orc.init_state(cfg, seed=seed), strict=True)
    s.trainer.eng.pack_weights(s.trainer.P, need_dgrad=True)
    return s


def _step(tr, x, eps):
    tr.step(x, 1.0, eps=eps)
    torch.cuda.synchronize()
    tr.eng.check_tc_status()
    return tr.opt.flat_g.clone(), tr.opt.flat_p.clone(), tr.report.clone()


# (kind, precision, B, env, T).  The segment length decides which kernels a step runs (tests/test_step_routes_host.py
# lists the routes of every length): at T = 128 the longest layer has 128 frames, every forward block runs fused, every
# weight gradient on the tensor cores, every norm backward in the cached kernel.  The other lengths reach the rest: the
# plain conv + avc_norm_apply_fwd forward (tf32 above 144 frames, fp32 above 256), the plain norm backward (above 128),
# the FFMA weight gradient inside a TF32 step (a layer above 128 frames, or a stride-2 one above 64, or one whose length
# is not a multiple of 8), the FFMA data gradient + avc_fold_add_fwd (a padded length above 256, the stride-2 parity
# data gradient above 512).
TRAIN_CASES = [("c80", "fp32", 8, {}, 128), ("c80", "tf32", 8, {}, 128), ("c512", "fp32", 8, {}, 128),
               ("c512", "tf32", 8, {}, 128), ("sn", "fp32", 8, {}, 128), ("sn", "tf32", 8, {}, 128),
               ("c80", "tf32", 37, {}, 128)] + [
    ("c80", "tf32", 8, {k: v}, 128) for k, v in (("AVC_FUSED_DENSE", "0"), ("AVC_FOLD_FUSED", "0"), ("AVC_NORM_BWD_FUSED", "1"),
                                                 ("AVC_WGRAD_ACC", "1"), ("AVC_WGRAD_STREAM", "0"), ("AVC_WGRAD_STREAM", "1"),
                                                 ("AVC_OVERLAP", "0"))] + [
    ("c80", p, 8, {}, T) for T in (64, 200, 256) for p in ("fp32", "tf32")] + [
    ("c512", "tf32", 8, {}, 256), ("sn", "tf32", 8, {}, 256), ("c80", "fp32", 4, {}, 512), ("c80", "tf32", 4, {}, 512)]


def _config(kind):
    return sn_config(80) if kind == "sn" else orc.default_config(80 if kind == "c80" else 512)


def _report(tag, chk):
    print(f"\n[{tag}] worst:", {k: f"{v:.2e} ({chk.where[k]})" for k, v in sorted(chk.worst.items())}, "ambiguous:", chk.amb)


@pytest.mark.parametrize("kind,precision,B,env,T", TRAIN_CASES,
                         ids=[f"{k}-{p}-B{b}" + "".join(f"-{n}={v}" for n, v in e.items()) + ("" if T == 128 else f"-T{T}")
                              for k, p, b, e, T in TRAIN_CASES])
def test_training_step_layers(monkeypatch, kind, precision, B, env, T):
    monkeypatch.setenv("AVC_PRECISION", precision)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    cfg = _config(kind)
    g = torch.Generator().manual_seed(11)
    x = torch.randn((B, cfg["SpeakerEncoder"]["c_in"], T), generator=g).cuda()
    eps = torch.randn((B, cfg["ContentEncoder"]["c_out"], T // 8), generator=g).cuda()

    plain = _step(_solver(cfg, B).trainer, x, eps)

    s = _solver(cfg, B)
    tr = s.trainer
    sn_names = tr.eng.sn_names()
    sn0 = {n: tuple(tr.P[n + sfx].clone() for sfx in (".weight_orig", ".weight_u", ".weight_v")) for n in sn_names}
    P = {k: v.clone() for k, v in tr.P.items()}     # the parameters the step reads (it updates them)
    cap = Capture()
    install(monkeypatch, tr.eng, cap)
    inst = _step(tr, x, eps)
    for a, b, what in zip(plain, inst, ("gradients", "parameters", "losses")):
        if env.get("AVC_WGRAD_ACC") == "1" or env.get("AVC_NORM_BWD_FUSED") == "1":
            # the two opt-in paths accumulate with atomics: equal up to the order of fp32 additions
            # (Adam normalises the gradient, so the parameters differ by more: measured 3.2e-5 of their largest)
            assert float((a - b).abs().max()) <= 2e-4 * float(a.abs().max()), f"the instrumented step changed the {what}"
        else:
            assert torch.equal(a.view(torch.int32), b.view(torch.int32)), f"the instrumented step changed the {what}"

    # with sn: W_bar as the engine read it, and its gradient before the spectral-norm backward
    G = dict(tr.G)
    for n in sn_names:
        P[n + ".weight"], G[n + ".weight"] = cap.sn[n]
    chk = Checker(cap, G, cfg, precision == "tf32")
    mu, ls, emb, dec, acts = LR.ae_forward(P, cfg, x, eps, chk, cap.tc)
    LR.ae_backward(P, cfg, x, eps, mu, ls, dec, acts, 1.0, chk, cap.tc)
    loss_rec, loss_kl, _ = tr._decode_report(inst[2].tolist())
    lr_, lk_, _, _, _ = LR.loss_grads(cfg, x, mu, ls, dec, 1.0)
    chk.err("misc", "loss_rec", abs(loss_rec - float(lr_)) / float(lr_))
    chk.err("misc", "loss_kl", abs(loss_kl - float(lk_)) / float(lk_))
    for n in sn_names:
        w0, u0, v0 = sn0[n]
        wbar, u1, v1, sigma = LR.sn_wbar(w0, u0, v0)
        chk.err("misc", n + ".W_bar", Checker._rel(cap.sn[n][0], wbar, wbar.abs().max()))
        ref = LR.sn_bwd(cap.sn[n][1], wbar, u1, v1, sigma)
        chk.err("grad", n + ".weight_orig", Checker._rel(tr.G[n + ".weight_orig"], ref, ref.abs().max()))
        chk.checked[n + ".weight_orig"] += 1
    _report(f"{kind} {precision} B={B} T={T} {env}", chk)

    names = set(tr.G)    # (with sn also name + ".weight": the gradient of W_bar, checked by its layer)
    assert {k for k, v in chk.checked.items() if v} == names, sorted(names ^ {k for k, v in chk.checked.items() if v})
    assert all(chk.checked[k] == 1 for k in names), {k: v for k, v in chk.checked.items() if v != 1}
    layers = {n for n in tr.eng.conv_names()}
    stray = [(n, t) for n, t in cap.launches if n in CONV_FAMILY and (t is None or t[0] not in layers)]
    assert not stray, stray[:5]
    assert not chk.problems, chk.problems[:10]
    tol = TOL[precision]
    bad = {k: (v, chk.where[k]) for k, v in chk.worst.items() if not v <= tol[k]}
    assert not bad, bad


def test_training_step_rejects_a_length_the_decoder_does_not_reproduce():
    """244 frames decode to 248: the loss would pair misaligned frames and read past x.  The step refuses before its
    first launch."""
    from adaptive_voice_conversion_b200 import _lib as L
    tr = _solver(_config("c80"), 2).trainer
    x = torch.randn((2, 80, 244), generator=torch.Generator().manual_seed(3)).cuda()
    torch.cuda.synchronize()
    n0 = L.launch_count()
    with pytest.raises(L.AvcError, match="T = 244 frames decodes to 248"):
        tr.step(x, 1.0)
    assert L.launch_count() == n0


# ------------------------------------------------------------------ inference
INFER_CASES = [(17, 9), (145, 600), (1000, 333)]


def eval_wbar(m, cap, chk):
    """W_bar of every spectral-norm layer as the engine computed it for a model in eval() (no power iteration: the
    stored u and v), checked against the float64 restatement -> {name + ".weight": W_bar} for the reference chain.
    The stored u and v are not W's singular vectors, so sigma = u^T W v may cancel: the error is measured against the
    magnitude of its terms, sum |u_i W_ij v_j| / |sigma| times W_bar's largest."""
    from _sn_ref import power_iteration64
    P, bufs = dict(m.named_parameters()), dict(m.named_buffers())
    wbar = {}
    for n, (w, iterate) in cap.wbar.items():
        if iterate:
            chk.problems.append(f"{n}: the spectral norm of an eval() model iterated u and v")
        w0, u, v = P[n + ".weight_orig"].detach(), bufs[n + ".weight_u"].double(), bufs[n + ".weight_v"].double()
        ref = power_iteration64(w0, u, v, iterate=False)[3]
        wm = w0.double().reshape(w0.shape[0], -1)
        cancel = float(u.abs() @ wm.abs() @ v.abs()) / abs(float(u @ wm @ v))
        chk.err("misc", n + ".W_bar", Checker._rel(w, ref, ref.abs().max() * cancel))
        wbar[n + ".weight"] = w
    return wbar


def inference_model(kind):
    """-> (AE on cuda in eval(), config).  eval() as a converter runs the model: with Decoder.sn, W_bar then comes
    from the stored u and v without a power iteration (torch's default init and its u and v: the oracle's init_state
    has no spectral norm)."""
    from adaptive_voice_conversion_b200.model import AE
    cfg = _config(kind)
    torch.manual_seed(0)
    m = AE(cfg)
    if kind != "sn":
        m.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
    return m.cuda().eval(), cfg


def inference_layers(monkeypatch, kind, precision, T, T_c):
    """Every layer of an unpadded AE.inference of 3 pairs (T source and T_c reference frames)."""
    monkeypatch.setenv("AVC_PRECISION", precision)
    monkeypatch.setenv("AVC_INFER_GRAPH", "0")
    m, cfg = inference_model(kind)
    g = torch.Generator().manual_seed(5)
    x = torch.randn((3, cfg["SpeakerEncoder"]["c_in"], T), generator=g).cuda()
    xc = torch.randn((3, cfg["SpeakerEncoder"]["c_in"], T_c), generator=g).cuda()
    m.inference(x, xc)            # packs the weights
    eng = m.engine(x.device)
    cap = Capture()
    install(monkeypatch, eng, cap)
    dec = m.inference(x, xc)
    torch.cuda.synchronize()
    eng.check_tc_status()
    P = dict(m.named_parameters())
    chk = Checker(cap, {}, cfg, precision == "tf32")
    assert set(cap.wbar) == set(eng.sn_names())
    P.update(eval_wbar(m, cap, chk))
    ref, _ = LR.ae_inference(P, cfg, x, xc, chk, cap.tc)
    chk.err("misc", "dec", Checker._rel(dec, ref, ref.abs().max()))
    _report(f"inference {kind} {precision} T={T} T_c={T_c}", chk)
    paths = {n for n, _ in cap.launches}
    print("entry points:", sorted(p for p in paths if p in CONV_FAMILY or "norm_apply" in p))
    assert len(cap.fwd) == len(eng.conv_names())
    assert not chk.problems, chk.problems[:10]
    tol = dict(TOL[precision])
    if precision == "tf32" and T < 32:
        # the decoder's in_conv normalises 3 latent frames here, and one row has |mean| / std = 80.  The fused tensor-core
        # epilogue takes the variance in one pass (E[c^2] - mean^2, csrc/conv_tc2.cu), which loses (mean / std)^2 * 2^-24
        # = 3.8e-4 of it to cancellation: measured 3.8e-4 (c512 5.5e-5, sn 1.6e-4).  The same case in fp32 (FFMA kernels)
        # stays at 5.5e-6 (c512 1.1e-5).
        tol["fwd"] = 1.2e-3
    bad = {k: (v, chk.where[k]) for k, v in chk.worst.items() if not v <= tol[k]}
    assert not bad, bad


@pytest.mark.parametrize("precision", ["fp32", "tf32"])
@pytest.mark.parametrize("T,T_c", INFER_CASES)
def test_inference_layers(monkeypatch, precision, T, T_c):
    inference_layers(monkeypatch, "c80", precision, T, T_c)
