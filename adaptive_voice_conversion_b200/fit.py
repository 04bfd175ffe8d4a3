"""Fit banked speaker codes: optimise each speaker's code on that speaker's recordings with the whole model frozen.

Trainable values: the codes only, float32 [S, c_out], each starting at the speaker's ``build_bank`` code over the same
utterances.  Every model parameter and every state_dict entry keeps its bits and the weight packs are never rebuilt,
so the result is still a bank: one [S, c_out] tensor that works with the one shared model (``-speaker``, mixes,
``evaluate.py -bank``).  The decoder reads a code only through its AdaIN affine layers.

Objective of speaker s: lambda_rec x the mean |dec - x| over s's crops, the segment_size-frame windows at every valid
start of each of the speaker's clips (``adapt.crop_index``).  dec is the conversion path -- the content encoder's mean
z = mu, no noise, eval mode -- so a code is fitted to the very function inference runs with it (and that
``adapt.heldout_rec`` scores).  With ``Decoder.sn`` the decoder uses its eval-mode W_bar: the stored u and v, no power
iteration and no spectral-norm backward.

One step of a wave (``CodeFitTrainer``) of S_w speakers x m crops each, B = S_w m, slot b reading code b div m:
gather the crops (``avc_segment_gather`` over the wave's order table, outside the graph); ``content_fwd(train=False)``
and z = mu; the decoder forward with its activations saved, the AdaIN rows computed from the expanded per-slot codes;
the grouped L1 loss and its gradient written straight into A4 (``avc_group_l1``); the decoder's backward with data
gradients only, down to demb [B, c_out] (``Engine.decoder_bwd(need_wgrad=False)``); one ``avc_code_adam``.

Update of code s: clip_grad_norm_ + Adam(amsgrad, weight_decay) applied to that code alone, in ``avc_adam_step``'s
order and formulas: g_s = the sum of its m demb rows (``avc_bias_grad``'s order), the clip coefficient
min(1, max_norm / (||g_s|| + 1e-6)), L2 decay, Adam.  Hyper-parameters are the config's ``optimizer`` section,
``lr`` overriding the rate.

Independence: every loss, clip and moment is per code, and each speaker's crop order is seeded by (seed, speaker name)
only (``speaker_seed``).  So a fitted code does not depend on which speakers share its wave or on the wave size:
batching speakers is a speed-up only.  Waves are consecutive chunks of the fittable speakers in bank order; a smaller
last wave is its own graph shape.  Each wave uploads its own speakers' clips only (``DeviceSegments``' layout).

A speaker with fewer than m crops (including one without a clip of segment_size frames) keeps its pooled code and is
listed as ``unfitted``.

A fitted bank records the run (``fitted``: steps, settings and ``model_fingerprint``, a sha256 of the content encoder,
the decoder and their config sections): a fitted code is tuned to that decoder, so ``SpeakerBank.load`` refuses it
against any other.  Fitted codes may drift from the speaker encoder's embedding space, so speaker identification
against a fitted bank (``evaluate.py -spk -bank``) measures something other than it does for pooled codes.
"""
from __future__ import annotations

import hashlib
import json
from typing import Callable, Dict, List, Mapping, Optional, Sequence

import numpy as np
import torch
import torch.nn as nn

from . import _lib as L
from .adapt import _host, crop_index, heldout_rec
from .data_utils import DeviceSegments, SegmentSampler
from .engine import A4
from .optim import FusedAdam
from .trainer import FusedTrainer

FORMAT = "avc-fit-1"
LOG_EVERY = 100


def model_fingerprint(model) -> str:
    """sha256 (hex) of what a fitted code is tuned to: every state_dict entry of the content encoder, then of the
    decoder, in key order (name, shape, float32 bytes), then their config sections as sorted JSON."""
    h = hashlib.sha256()
    for prefix in ("content_encoder.", "decoder."):
        for name, t in model.state_dict().items():
            if name.startswith(prefix):
                h.update(name.encode())
                h.update(json.dumps(list(t.shape)).encode())
                h.update(t.detach().to(device="cpu", dtype=torch.float32).contiguous().numpy().tobytes())
    h.update(json.dumps([model.config["ContentEncoder"], model.config["Decoder"]], sort_keys=True).encode())
    return h.hexdigest()


# ----------------------------------------------------------------------------- schedule (host only)
def speaker_seed(seed: int, name: str) -> int:
    """The crop-order seed of one speaker: 63 bits of sha256("<seed>/<name>"), a function of the run's seed and the
    speaker's name only."""
    return int.from_bytes(hashlib.sha256(f"{int(seed)}/{name}".encode()).digest()[:8], "little") & ((1 << 63) - 1)


def speaker_order(n_crops: int, m: int, steps: int, seed: int, name: str) -> np.ndarray:
    """int64 [steps, m]: the entries (0 .. n_crops - 1 of the speaker's crop index) its m slots hold at each step --
    SegmentSampler(n_crops, m, seed=speaker_seed(seed, name), drop_last=True)'s batches, one per step."""
    smp = SegmentSampler(n_crops, m, seed=speaker_seed(seed, name), drop_last=True)
    out = np.empty((steps, m), np.int64)
    for k in range(steps):
        epoch, first, _ = smp.locate(k)
        out[k] = smp.order(epoch)[first:first + m].numpy()
    return out


def plan_waves(speakers: Sequence[str], per_wave: int) -> List[List[str]]:
    """Consecutive chunks of per_wave speakers, in the given (bank) order; the last one may be smaller."""
    if per_wave < 1:
        raise ValueError(f"speakers per wave must be >= 1 (got {per_wave})")
    speakers = list(speakers)
    return [speakers[i:i + per_wave] for i in range(0, len(speakers), per_wave)]


def order_table(n_crops: Sequence[int], m: int, steps: int, seed: int, names: Sequence[str]) -> np.ndarray:
    """int32 [steps * S_w * m]: a wave's gather order.  Position (k S_w + s) m + j holds speaker s's speaker_order
    entry (k, j), offset by the crops of the speakers before s in the wave's index."""
    off = np.concatenate([[0], np.cumsum(n_crops)[:-1]]).astype(np.int64)
    tab = np.stack([speaker_order(n, m, steps, seed, s) + o for n, o, s in zip(n_crops, off, names)], axis=1)
    return np.ascontiguousarray(tab.reshape(-1), dtype=np.int32)


def plan(bank_speakers: Sequence[str], bank_utterances: Sequence[Sequence[str]], lengths: Mapping[str, int],
         segment_size: int, m: int):
    """{speaker: {"index", "used", "skipped", "n_crops"}} (adapt.crop_index over the speaker's bank utterances in bank
    order) and the unfitted speakers (fewer than m crops), in bank order."""
    per, unfitted = {}, []
    for s, us in zip(bank_speakers, bank_utterances):
        index, used, skipped = crop_index({u: int(lengths[u]) for u in us}, segment_size)
        per[s] = {"index": index, "used": used, "skipped": skipped, "n_crops": len(index)}
        if len(index) < m:
            unfitted.append(s)
    return per, unfitted


# ----------------------------------------------------------------------------- the step
class _Codes(nn.Module):
    def __init__(self, codes: torch.Tensor):
        super().__init__()
        self.codes = nn.Parameter(codes.detach().to(torch.float32).contiguous().clone())
        self._flat = None

    def flatten_parameters(self) -> torch.Tensor:
        self._flat = self.codes.data.view(-1)
        return self._flat


class CodeAdam(FusedAdam):
    """FusedAdam's buffers and hyper-parameter vector over the codes [S, c_out]; one step counter per code.  There is
    no model gradient: named_grad_views gives None (FusedTrainer then registers no gradient buffer)."""

    def __init__(self, codes: _Codes, **kw):
        super().__init__(codes, **kw)
        self.steps = torch.zeros(codes.codes.shape[0], dtype=torch.float32, device=self.flat_p.device)

    def named_grad_views(self, model):
        return None

    def step(self, closure=None):
        raise L.AvcError("CodeAdam: the codes are updated by avc_code_adam (CodeFitTrainer._update)")


class CodeFitTrainer(FusedTrainer):
    """FusedTrainer's step machinery (CUDA-graph capture on the third step of a shape and replay, AVC_GRAPH=0 eager,
    the 16-byte report block, losses_async) around the fitting step of the module docstring, for waves of S speakers x
    m crops.  ``codes`` [S, c_out] are the trained values; ``reset(codes)`` starts a new wave of the same shape (the
    captured graph keeps its buffers).  The report block's loss_rec is the batch's mean L1; loss_kl and grad_norm are
    0 (the per-code norms are ``gnorm``).  ``gsum`` (float64 [S]) holds each code's L1 sum of the last step."""

    def __init__(self, model, config: dict, S: int, m: int, lr=None):
        o = config["optimizer"]
        dev = next(model.parameters()).device
        c_out = int(config["SpeakerEncoder"]["c_out"])
        if S < 1 or m < 1:
            raise ValueError(f"CodeFitTrainer: need S >= 1 and m >= 1 (got {S}, {m})")
        if c_out % 4 != 0 or c_out > L.CODE_MAX_C:
            raise L.AvcError(f"code fitting supports c_out a multiple of 4 up to {L.CODE_MAX_C} (got {c_out})")
        self.S, self.m, self.B = int(S), int(m), int(S) * int(m)
        self._mod = _Codes(torch.zeros(S, c_out, device=dev))
        opt = CodeAdam(self._mod, lr=o["lr"] if lr is None else float(lr), betas=(o["beta1"], o["beta2"]),
                       amsgrad=o["amsgrad"], weight_decay=o["weight_decay"], max_norm=o["grad_norm"])
        self.codes = self._mod.codes.data
        self.grad = opt.flat_g.view(S, c_out)            # g_s of the last step, before clipping
        self.gnorm = torch.zeros(S, dtype=torch.float32, device=dev)
        self.gsum = torch.zeros(S, dtype=torch.float64, device=dev)
        self._part = torch.zeros(self.B, dtype=torch.float64, device=dev)
        self.emb = torch.zeros(self.B, c_out, dtype=torch.float32, device=dev)
        super().__init__(model, opt, config)
        if self.sn:   # eval-mode W_bar from the stored u and v, packed once
            self.eng.spectral_norm(self.P, iterate=False)
            self.eng.pack_weights(self.P, need_dgrad=True, prefixes=("decoder.",))
        dl = config["data_loader"]
        self._x = torch.empty(self.B, int(config["ContentEncoder"]["c_in"]), int(dl["segment_size"]), device=dev)
        self._demb = None

    def reset(self, codes: torch.Tensor):
        """Start a wave: the codes [S, c_out], zero moments and step counters, the expanded rows of the first step."""
        with torch.no_grad():
            self.codes.copy_(codes.reshape(self.S, -1))
            for t in (self.opt.flat_m, self.opt.flat_v, self.opt.flat_vmax, self.opt.steps, self.grad, self.gnorm):
                t.zero_()
            self.emb.copy_(self.codes.repeat_interleave(self.m, dim=0))

    def _fwd_bwd(self, x: torch.Tensor, eps):
        eng, P = self.eng, self.P
        mu4, ls4, _ = eng.content_fwd(P, x, False)
        _, _, z4 = eng.reparam_fwd(mu4, ls4, None, want_planar=False)   # z = mu, as the conversion path
        dec4, cd = eng.decoder_fwd(P, z4, self.emb, True)
        ddec4 = A4.empty(dec4.B, dec4.C, dec4.T, self.dev)
        self.n_rec, self.n_lat = dec4.B * dec4.C * dec4.T, 1
        rnd = eng.precision == "tf32" and not eng.fwd_fp32   # avc_pack_a4's rounding of a gradient operand
        d = L.GroupL1Desc(B=dec4.B, C=dec4.C, T=dec4.T, m=self.m, round_tf32=int(rnd), dec=dec4.ptr, x=x.data_ptr(),
                          hp=self.opt.hp.data_ptr(), ddec=ddec4.ptr, part=self._part.data_ptr(),
                          sums=self.gsum.data_ptr(), total=self.sums.data_ptr())
        L.check(self.lib.avc_group_l1(d, eng.stream), "avc_group_l1")
        ddec4.tf32 = rnd
        _, self._demb = eng.decoder_bwd(P, None, cd, ddec4, need_dz=False, need_wgrad=False)
        return None

    def _update(self):
        o = self.opt
        d = L.CodeAdamDesc(S=self.S, m=self.m, C=self.codes.shape[1], demb=self._demb.data_ptr(),
                           codes=self.codes.data_ptr(), exp_avg=o.flat_m.data_ptr(), exp_avg_sq=o.flat_v.data_ptr(),
                           max_exp_avg_sq=o.flat_vmax.data_ptr(), steps=o.steps.data_ptr(), grad=self.grad.data_ptr(),
                           gnorm=self.gnorm.data_ptr(), emb=self.emb.data_ptr(), hp=o.hp.data_ptr())
        L.check(self.lib.avc_code_adam(d, self.eng.stream), "avc_code_adam")

    def run_step(self, corpus: "WaveCorpus", k: int):
        """Step k of the wave: gather its crops into the step's input buffer (the captured graph's own once there is
        one, so a replay copies nothing), then step."""
        x = self._static if self._graphs is not None else self._x
        corpus.gather(x, k * self.B, self.B)
        self.step(x, 0.0)


class WaveCorpus:
    """The clips of one wave's speakers on the device (DeviceSegments' frames and start table) and the wave's order
    table for all its steps (order_table), uploaded once."""

    def __init__(self, mels: Mapping[str, object], index, order: np.ndarray, config: dict, device):
        dl = config["data_loader"]
        used = list(dict.fromkeys(u for u, _ in index))
        self.ds = DeviceSegments({u: _host(mels[u]) for u in used}, index, int(dl["segment_size"]), 1, 1,
                                 int(config["ContentEncoder"]["c_in"]), device=device)
        self.order = torch.from_numpy(order).to(device)

    def gather(self, x: torch.Tensor, first: int, count: int):
        if first < 0 or first + count > self.order.numel():
            raise ValueError(f"WaveCorpus.gather: entries [{first}, {first + count}) of a table of {self.order.numel()}")
        ds = self.ds
        d = L.GatherDesc(corpus=ds.corpus.data_ptr(), starts=ds.starts.data_ptr(), order=self.order.data_ptr(),
                         x=x.data_ptr(), first=first, batch=count, seg=ds.segment_size, frame=1, n_mels=ds.n_mels)
        L.check(ds.lib.avc_segment_gather(d, torch.cuda.current_stream(x.device).cuda_stream), "avc_segment_gather")


# ----------------------------------------------------------------------------- the run
def fit_wave(trainer: CodeFitTrainer, corpus: WaveCorpus, codes0: torch.Tensor, steps: int,
             log_every: int = LOG_EVERY):
    """`steps` steps of one wave from codes0 [S, c_out]; returns (codes [S, c_out], log) with log = [(step, L1 sums
    float64 [S], pre-clip norms [S])] of the first step, every log_every-th and the last, read once at the end (device
    copies, so the host never waits inside the loop)."""
    trainer.reset(codes0)
    snaps = []
    for k in range(steps):
        trainer.run_step(corpus, k)
        if k % log_every == 0 or k == steps - 1:
            snaps.append((k, trainer.gsum.clone(), trainer.gnorm.clone()))
    trainer.eng.check_tc_status()
    return trainer.codes.clone(), [(k, s.cpu().numpy(), g.cpu().numpy()) for k, s, g in snaps]


def fit_bank(model, bank, mels: Mapping[str, object], steps: int, lr=None, crops: int = 8, speakers_per_wave: int = 16,
             seed: int = 0, heldout: Optional[Mapping[str, Mapping[str, object]]] = None,
             mcd: Optional[Callable] = None, log_every: int = LOG_EVERY):
    """Fit every code of `bank` (a SpeakerBank of `model`) on its speaker's bank utterances `mels` ({id:
    attr-normalised [T, n_mels]}); returns (the fitted SpeakerBank, the report).  heldout {speaker: {id: mel}}: scored
    before (pooled code) and after (fitted code) with adapt.heldout_rec.  mcd(model, {speaker: code}) -> evaluate_mcd's
    dict: a second held-out measure over the fitted speakers at once, before and after.  `model` is not modified."""
    from .speaker_bank import SpeakerBank
    cfg = model.config
    if int(cfg["data_loader"]["frame_size"]) != 1:
        raise ValueError(f"code fitting supports data_loader.frame_size 1 only (got {cfg['data_loader']['frame_size']})")
    if steps < 1 or crops < 1 or speakers_per_wave < 1:
        raise ValueError(f"need steps, crops and speakers per wave >= 1 (got {steps}, {crops}, {speakers_per_wave})")
    dev = next(model.parameters()).device
    seg = int(cfg["data_loader"]["segment_size"])
    lam = float(cfg["lambda"]["lambda_rec"])
    per, unfitted = plan(bank.speakers, bank.utterances, {u: int(mels[u].shape[0]) for u in bank.utterance_ids()},
                         seg, crops)
    fittable = [s for s in bank.speakers if s not in unfitted]
    waves = plan_waves(fittable, speakers_per_wave)
    codes = bank.codes.detach().clone()
    pooled = {s: codes[bank.index(s)].clone() for s in bank.speakers}
    before_rec = {s: heldout_rec(model, heldout[s], pooled[s]) for s in bank.speakers if heldout and s in heldout}
    before_mcd = mcd(model, {s: pooled[s] for s in fittable}) if mcd is not None and fittable else None
    trainers: Dict[int, CodeFitTrainer] = {}
    logs: Dict[str, list] = {}
    wave_of: Dict[str, int] = {}
    for w, names in enumerate(waves):
        S = len(names)
        if S not in trainers:
            trainers[S] = CodeFitTrainer(model, cfg, S, crops, lr)
        tr = trainers[S]
        index = [e for s in names for e in per[s]["index"]]
        order = order_table([per[s]["n_crops"] for s in names], crops, steps, seed, names)
        corpus = WaveCorpus(mels, index, order, cfg, dev)
        rows = torch.stack([pooled[s] for s in names]).to(dev)
        fitted, log = fit_wave(tr, corpus, rows, steps, log_every)
        del corpus
        n_frames = crops * int(cfg["ContentEncoder"]["c_in"]) * seg
        for i, s in enumerate(names):
            codes[bank.index(s)] = fitted[i]
            wave_of[s] = w
            logs[s] = [{"step": int(k), "loss_rec": float(lam * sums[i] / n_frames), "grad_norm": float(gn[i])}
                       for k, sums, gn in log]
    after_rec = {s: heldout_rec(model, heldout[s], codes[bank.index(s)]) for s in before_rec}
    after_mcd = mcd(model, {s: codes[bank.index(s)] for s in fittable}) if before_mcd is not None else None
    tr0 = next(iter(trainers.values()), None)
    o = cfg["optimizer"]
    settings = {"steps": int(steps), "lr": float(o["lr"] if lr is None else lr), "crops": int(crops),
                "speakers_per_wave": int(speakers_per_wave), "seed": int(seed), "segment_size": seg,
                "betas": [float(o["beta1"]), float(o["beta2"])], "weight_decay": float(o["weight_decay"]),
                "grad_norm": float(o["grad_norm"]), "amsgrad": bool(o["amsgrad"]), "lambda_rec": lam,
                "precision": model.engine(dev).precision}
    record = dict(settings, model_fingerprint=model_fingerprint(model), fitted=list(fittable))
    out = SpeakerBank(bank.speakers, codes, bank.n_utts, bank.utterances, bank.fingerprint, bank.n_skipped,
                      fitted=record, pitch=bank.pitch)     # pitch profiles describe the recordings, not the codes
    speakers = {}
    for s in bank.speakers:
        p = per[s]
        held = None
        if s in before_rec or before_mcd is not None:
            held = {"before": {}, "after": {}}
            if s in before_rec:
                held["before"]["rec"], held["after"]["rec"] = before_rec[s], after_rec[s]
            if before_mcd is not None and s in fittable:
                held["before"]["mcd"] = before_mcd["speakers"].get(s)
                held["after"]["mcd"] = after_mcd["speakers"].get(s)
        speakers[s] = {"fitted": s in wave_of, "wave": wave_of.get(s),
                       "clips": {"used": list(p["used"]), "skipped": list(p["skipped"]), "n_crops": int(p["n_crops"])},
                       "losses": logs.get(s, []), "heldout": held}
    report = make_report(settings, unfitted, speakers, len(waves),
                         tr0.launches_per_step if tr0 is not None else 0,
                         {"before": before_mcd, "after": after_mcd} if before_mcd is not None else None)
    return out, report


REPORT_KEYS = ("format", "settings", "precision", "unfitted", "n_waves", "launches_per_step", "mcd", "speakers")
SPEAKER_KEYS = ("fitted", "wave", "clips", "losses", "heldout")


def make_report(settings, unfitted, speakers, n_waves, launches, mcd) -> dict:
    """The JSON document of a run: {"format", "settings", "precision", "unfitted": [speakers kept at their pooled
    code], "n_waves", "launches_per_step" (of the step graph, the crop gather not counted), "mcd": {"before", "after"}
    (evaluate_mcd's run-level results) or null, "speakers": {name: {"fitted", "wave", "clips": {"used", "skipped",
    "n_crops"}, "losses": [{"step", "loss_rec", "grad_norm"}], "heldout": {"before", "after"} or null}}}.  before /
    after map a measure ("rec": heldout_rec's dict, "mcd": the speaker's evaluate_mcd entry) to its result."""
    return {"format": FORMAT, "settings": dict(settings), "precision": settings["precision"], "unfitted": list(unfitted),
            "n_waves": int(n_waves), "launches_per_step": int(launches), "mcd": mcd,
            "speakers": {s: {k: v[k] for k in SPEAKER_KEYS} for s, v in speakers.items()}}
