"""Held-out evaluation: the reconstruction and KL losses of the conversion path on the sets preprocess.py writes
(``in_test``: seen speakers, unseen utterances; ``out_test``: unseen speakers), or preprocess_libri.py (``dev``: held
out of the training subset; ``test``: the test subset).

For a set S (``<S>.pkl`` and its index ``<S>_samples_<segment_size>.json``) every index entry i is cut into a segment
x_i exactly as ``DeviceSegments`` cuts a training batch, and

    dec_i = AE.inference(x_i, x_i)        (content mean, the speaker of the same segment, no noise)
    rec_i = sum |dec_i - x_i|,   kl_i = sum (exp(ls_i) + mu_i^2 - 1 - ls_i)      (float64, avc_eval_losses)
    loss_rec = sum_i rec_i / (n C T),   loss_kl = 0.5 sum_i kl_i / (n C_lat T_lat)

(mu_i, ls_i: the content encoder's outputs).  These are the training losses without the lambda weights, the KL
annealing and the sampled z, so values from different iterations, checkpoints and configs compare.  The model runs in
eval mode (Decoder.sn: the stored u and v, no power iteration) and no random number is drawn.

Under data parallelism batch j of a set goes to rank j mod world.  Every segment then sits in the batch it has with one
GPU, each table row is written by one rank and is zero on the others, and one all_reduce(SUM) of the float64 table is
exact: the results are the same bits for any world size.
"""
from __future__ import annotations

import os
from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from .data_utils import DeviceSegments, check_segment_size, corpus_device_bytes, load_corpus, validate_corpus
from .utils import local_device


def rank_batches(n: int, batch_size: int, rank: int = 0, world: int = 1) -> List[Tuple[int, int]]:
    """(first entry, count) of the batches of an n-entry set that `rank` evaluates: batch j covers entries
    [j B, min(n, (j + 1) B)) and belongs to rank j mod world."""
    if n < 1 or batch_size < 1 or world < 1 or not 0 <= rank < world:
        raise ValueError(f"rank_batches: need n, batch_size, world >= 1 and 0 <= rank < world "
                         f"(n={n}, batch_size={batch_size}, rank={rank}, world={world})")
    return [(f, min(batch_size, n - f)) for j, f in enumerate(range(0, n, batch_size)) if j % world == rank]


def speaker_of(utt_id: str) -> str:
    """The speaker of an utterance id: everything up to its first '_'.  VCTK: p225_001.wav -> p225; LibriTTS
    (<speaker>_<chapter>_<paragraph>_<sentence>.wav): 103_1241_000000_000001.wav -> 103."""
    return str(utt_id).split("_", 1)[0]


def reduce_table(table: np.ndarray, n_rec: int, n_lat: int, rows=None) -> Dict[str, float]:
    """{loss_rec, loss_kl, n} of the rows `rows` (default: all) of a float64 [n][2] table of (rec_i, kl_i), added
    sequentially in index order; n_rec = C*T and n_lat = C_lat*T_lat elements per segment."""
    t = np.asarray(table, dtype=np.float64)
    if rows is not None:
        t = t[np.asarray(rows, dtype=np.int64)]
    n = len(t)
    rec, kl = (float(np.cumsum(t[:, j])[-1]) for j in (0, 1))
    return {"loss_rec": rec / (n * n_rec), "loss_kl": 0.5 * kl / (n * n_lat), "n": n}


def summarize(table: np.ndarray, utts: Sequence[str], n_rec: int, n_lat: int, per_speaker: bool = False) -> dict:
    """reduce_table over the whole set, plus {speaker: reduce_table over its entries} (in order of first appearance)
    under "speakers" when per_speaker."""
    res = reduce_table(table, n_rec, n_lat)
    if per_speaker:
        groups: Dict[str, List[int]] = {}
        for i, u in enumerate(utts):
            groups.setdefault(speaker_of(u), []).append(i)
        res["speakers"] = {s: reduce_table(table, n_rec, n_lat, rows) for s, rows in groups.items()}
    return res


def eval_params(model, device):
    """(engine, parameter dict) of `model` ready for Engine.eval_losses: the same tensors (and, with Decoder.sn, the same
    W_bar buffers) a FusedTrainer or AE.inference on this device reads, with the eval-mode weights prepared."""
    eng = model.engine(device)
    P = dict(model.named_parameters())
    if eng.sn_names():
        P.update(model.named_buffers())
        eng.bind_spectral_norm(P)
    eng.prepare_eval(P)
    return eng, P


def _set_paths(data_dir: str, name: str, segment_size: int):
    return os.path.join(data_dir, f"{name}.pkl"), os.path.join(data_dir, f"{name}_samples_{segment_size}.json")


class HeldOut:
    """The held-out sets `sets` of `data_dir`, resident on the device, and their evaluation.

    Construction loads and validates every set (a bad file raises validate_corpus's ValueError here, before any
    training step), then uploads them.  reserved_bytes: device memory already given to the training corpus; a
    ValueError naming the sizes is raised when it and the sets exceed 3/4 of the device's total memory."""

    def __init__(self, sets: Sequence[str], data_dir: str, config: dict, rank: int = 0, world: int = 1,
                 reserved_bytes: int = 0, total_memory: int = None, device=None):
        if not sets:
            raise ValueError("HeldOut: no evaluation set named")
        if data_dir in (None, "synthetic"):
            raise ValueError("held-out evaluation needs a data directory with the test sets (-d <data_dir>)")
        dl = config["data_loader"]
        check_segment_size(config)
        self.sets = list(sets)
        self.batch_size = int(dl["batch_size"])
        self.rank, self.world = rank, world
        self.dev = torch.device(device) if device is not None else local_device()
        c_in = config["ContentEncoder"]["c_in"]
        loaded, sizes = {}, {}
        for name in self.sets:
            data, index = load_corpus(*_set_paths(data_dir, name, dl["segment_size"]))
            _, n_mels, total = validate_corpus(data, index, dl["segment_size"], dl["frame_size"], c_in)
            loaded[name] = (data, index)
            sizes[name] = corpus_device_bytes(total, n_mels, len(index))
        if total_memory is None:
            total_memory = torch.cuda.get_device_properties(self.dev).total_memory
        need = reserved_bytes + sum(sizes.values())
        if need > total_memory * 3 // 4:
            raise ValueError("the device corpus and the evaluation sets need more than 3/4 of the device's "
                             f"{total_memory / 1e9:.1f} GB: training {reserved_bytes / 1e9:.2f} GB + "
                             + ", ".join(f"{s} {b / 1e9:.2f} GB" for s, b in sizes.items()))
        self.bytes = sizes
        self.data: Dict[str, DeviceSegments] = {}
        self.utts: Dict[str, List[str]] = {}
        for name in self.sets:
            data, index = loaded.pop(name)
            seg = DeviceSegments(data, index, dl["segment_size"], dl["frame_size"], self.batch_size, c_in, rank=0,
                                 shuffle=False, device=self.dev)
            seg.load_epoch(0)     # the index order
            self.data[name] = seg
            self.utts[name] = [u for u, _ in index]
            del data, index
        if rank == 0:
            print("evaluation sets: " + ", ".join(f"{s} {len(self.utts[s])} entries ({self.bytes[s] / 1e9:.2f} GB on the device)"
                                                  for s in self.sets))

    def tables(self, model) -> Dict[str, torch.Tensor]:
        """{set: float64 [n, 2] device table of (rec_i, kl_i)}, complete on every rank (all-reduced when world > 1)."""
        eng, P = eval_params(model, self.dev)
        out = {}
        for name in self.sets:
            seg = self.data[name]
            n = seg.sampler.n
            tab = torch.zeros((n, 2), dtype=torch.float64, device=self.dev)
            for first, count in rank_batches(n, self.batch_size, self.rank, self.world):
                eng.eval_losses(P, seg.gather(first, count), tab, first)
            if self.world > 1:
                torch.distributed.all_reduce(tab, op=torch.distributed.ReduceOp.SUM)
            out[name] = tab
        return out

    def evaluate(self, model, per_speaker: bool = False) -> dict:
        """{set: {"loss_rec", "loss_kl", "n"[, "speakers": {speaker: {...}}]}} of `model` (an AE on this device) as
        defined in the module docstring.  Collective under data parallelism: every rank calls it."""
        tabs = {s: t.cpu().numpy() for s, t in self.tables(model).items()}
        res = {}
        for name in self.sets:
            seg = self.data[name]
            n_rec = seg.c_in * seg.T
            n_lat = self._latent_elems(model, seg.T)
            res[name] = summarize(tabs[name], self.utts[name], n_rec, n_lat, per_speaker)
        return res

    @staticmethod
    def _latent_elems(model, T: int) -> int:
        """C_lat * T_lat of the content encoder's output for segments of T steps."""
        ce = model.config["ContentEncoder"]
        t = T
        for s in ce["subsample"][: ce["n_conv_blocks"]]:
            t = -(-t // s)
        return ce["c_out"] * t
