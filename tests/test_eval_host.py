"""CPU: the host side of the held-out evaluation.  The rank assignment of batches, the argument checks of
avc_eval_losses, the chunking of Solver.train around evaluations (with a fake run_steps), the host reduction and the
per-speaker grouping against a float64 restatement, the .eval.jsonl lines, and HeldOut's load-time errors."""
import ctypes
import json
import types

import numpy as np
import pytest

from _eval_data import write_data_dir
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import evaluate as E


@pytest.mark.parametrize("world", range(1, 9))
@pytest.mark.parametrize("n, B", [(1, 4), (64, 16), (70, 16), (100, 7), (10000, 128), (10000, 256)])
def test_rank_batches_cover_every_entry_once_in_the_single_gpu_batches(world, n, B):
    single = E.rank_batches(n, B, 0, 1)
    assert single[0][0] == 0 and sum(c for _, c in single) == n
    assert [c for _, c in single[:-1]] == [B] * (len(single) - 1)
    assert single[-1][1] == (n % B or B)          # short last batch when B does not divide n
    seen = np.zeros(n, dtype=np.int64)
    batches = []
    for r in range(world):
        mine = E.rank_batches(n, B, r, world)
        for j, (first, count) in enumerate(mine):
            seen[first:first + count] += 1
            assert single.index((first, count)) % world == r
        batches += mine
    assert (seen == 1).all()
    assert sorted(batches) == single              # every entry in the same batch as with one GPU


def test_rank_batches_rejects_bad_arguments():
    for args in [(0, 4, 0, 1), (4, 0, 0, 1), (4, 4, 1, 1), (4, 4, -1, 2), (4, 4, 0, 0)]:
        with pytest.raises(ValueError):
            E.rank_batches(*args)


def test_eval_losses_rejects_invalid_arguments_without_a_device():
    lib = L.load()
    fake = 0x10000     # never dereferenced: every case fails validation before a launch
    good = dict(B=4, C=80, T=128, C_lat=128, T_lat=16, dec=fake, x=fake, mu=fake, ls=fake, out=fake, first=0)
    cases = [({"dec": None}, "null pointer"), ({"x": None}, "null pointer"), ({"mu": None}, "null pointer"),
             ({"ls": None}, "null pointer"), ({"out": None}, "null pointer"), ({"B": 0}, "positive"), ({"C": -4}, "positive"),
             ({"T": 0}, "positive"), ({"C_lat": 0}, "positive"), ({"T_lat": -1}, "positive"), ({"C": 82}, "multiples of 4"),
             ({"C_lat": 126}, "multiples of 4"), ({"first": -1}, "first")]
    n0 = L.launch_count()
    for patch, msg in cases:
        rc = lib.avc_eval_losses(L.EvalDesc(**{**good, **patch}), None)
        assert rc == L.ERR_INVALID, patch
        assert msg in L.last_error(), (patch, L.last_error())
    assert lib.avc_eval_losses(None, None) == L.ERR_INVALID and "null descriptor" in L.last_error()
    assert L.launch_count() == n0


def test_eval_desc_layout_matches_the_header(tmp_path):
    import os
    import subprocess
    from conftest import ROOT
    c = tmp_path / "s.c"
    c.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "avc_b200.h"\nint main(){printf("%zu %zu %zu\\n", '
                 'sizeof(avc_eval_desc), offsetof(avc_eval_desc, dec), offsetof(avc_eval_desc, first));return 0;}\n')
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(tmp_path / "s")])
    sizes = [int(v) for v in subprocess.check_output([str(tmp_path / "s")]).split()]
    assert sizes == [ctypes.sizeof(L.EvalDesc), L.EvalDesc.dec.offset, L.EvalDesc.first.offset]


# ----------------------------------------------------------------------------- Solver.train chunking
def fake_solver(tmp_path, eval_steps, iteration=0, rank=0):
    from adaptive_voice_conversion_b200.config import default_config
    from adaptive_voice_conversion_b200.solver import Solver
    from adaptive_voice_conversion_b200.utils import Logger
    s = Solver.__new__(Solver)
    s.config = default_config(80)
    s.args = types.SimpleNamespace(summary_steps=1, save_steps=10 ** 9, tag="t", store_model_path=str(tmp_path / "m"),
                                   eval_steps=eval_steps)
    s.rank, s.world, s.iteration = rank, 1, iteration
    s.logger = Logger(str(tmp_path / "log"))
    s.calls = []

    def run_steps(n, lambda_of=None, on_step=None):
        s.calls.append(("run", s.iteration, n, [lambda_of(i) for i in range(s.iteration, s.iteration + n)]))
        s.iteration += n

    def evaluate(per_speaker=False):
        s.calls.append(("eval", s.iteration))
        return {"in_test": {"loss_rec": 0.5 + s.iteration, "loss_kl": 0.25, "n": 3}}
    s.run_steps, s.evaluate = run_steps, evaluate
    return s


def test_train_without_eval_steps_makes_one_run_steps_call(tmp_path):
    s = fake_solver(tmp_path, 0)
    s.train(25)
    assert [c[:3] for c in s.calls] == [("run", 0, 25)]
    assert not (tmp_path / "m.eval.jsonl").exists()


@pytest.mark.parametrize("start, n, k, ends", [
    (0, 25, 10, [10, 20, 25]), (0, 30, 10, [10, 20, 30]), (0, 5, 10, [5]), (0, 1, 1, [1]),
    (13, 20, 10, [20, 30, 33]), (13, 7, 10, [20]), (20, 10, 10, [30]), (7, 3, 4, [8, 10])])
def test_train_chunks_end_at_multiples_of_eval_steps_and_at_the_last_iteration(tmp_path, start, n, k, ends):
    s = fake_solver(tmp_path, k, iteration=start)
    ref = fake_solver(tmp_path / "ref", 0, iteration=start)
    s.train(n)
    ref.train(n)
    runs = [c for c in s.calls if c[0] == "run"]
    evals = [c[1] for c in s.calls if c[0] == "eval"]
    assert evals == ends
    assert [(c[1], c[1] + c[2]) for c in runs] == list(zip([start] + ends[:-1], ends))
    assert all(s.calls[2 * i][0] == "run" and s.calls[2 * i + 1][0] == "eval" for i in range(len(ends)))
    assert [lam for c in runs for lam in c[3]] == ref.calls[0][3]     # the same lambda schedule as one call
    lines = [json.loads(line) for line in (tmp_path / "m.eval.jsonl").read_text().splitlines()]
    assert [ln["iteration"] for ln in lines] == ends
    assert lines[0]["sets"]["in_test"] == {"loss_rec": 0.5 + ends[0], "loss_kl": 0.25, "n": 3}
    assert s.logger.last["t/eval_in_test"] == ({"loss_rec": 0.5 + ends[-1], "loss_kl": 0.25}, ends[-1])


def test_only_rank_0_logs(tmp_path):
    s = fake_solver(tmp_path, 5, rank=1)
    s.train(10)
    assert [c[1] for c in s.calls if c[0] == "eval"] == [5, 10]
    assert not (tmp_path / "m.eval.jsonl").exists() and not s.logger.last


# ----------------------------------------------------------------------------- host reduction
def test_reduction_and_speaker_grouping_match_a_float64_restatement():
    rng = np.random.default_rng(3)
    n, n_rec, n_lat = 1001, 80 * 128, 128 * 16
    tab = np.stack([rng.uniform(0, 1e4, n), rng.uniform(0, 3e3, n)], axis=1)
    utts = [f"p{225 + int(rng.integers(7))}_{i:03d}" for i in range(n)]
    utts[5] = "s5"   # an id without '_' is its own speaker
    res = E.summarize(tab, utts, n_rec, n_lat, per_speaker=True)

    def restate(rows):
        rec = kl = np.float64(0)
        for i in rows:
            rec += tab[i, 0]
            kl += tab[i, 1]
        return {"loss_rec": float(rec / (len(rows) * n_rec)), "loss_kl": float(0.5 * kl / (len(rows) * n_lat)), "n": len(rows)}
    assert {k: res[k] for k in ("loss_rec", "loss_kl", "n")} == restate(range(n))
    groups = {}
    for i, u in enumerate(utts):
        groups.setdefault(u.split("_")[0], []).append(i)
    assert list(res["speakers"]) == list(groups) and "s5" in groups
    for spk, rows in groups.items():
        assert res["speakers"][spk] == restate(rows), spk
    assert sum(r["n"] for r in res["speakers"].values()) == n
    assert E.speaker_of("p225_001") == "p225" and E.speaker_of("p225_001_mic2") == "p225"
    assert "speakers" not in E.summarize(tab, utts, n_rec, n_lat)
    json.loads(json.dumps(res))


# ----------------------------------------------------------------------------- HeldOut load-time errors
def test_held_out_rejects_bad_sets_before_touching_the_device(tmp_path):
    import pickle
    from adaptive_voice_conversion_b200.config import default_config
    cfg = default_config(80)
    d = write_data_dir(tmp_path / "data", 80, {"in_test": 20, "out_test": 10})
    with pytest.raises(ValueError, match="data directory"):
        E.HeldOut(["in_test"], "synthetic", cfg, device="cuda")
    with pytest.raises(ValueError, match="in_test .* out_test"):      # the sizes exceed 3/4 of a 1 MB device
        E.HeldOut(["in_test", "out_test"], d, cfg, total_memory=1 << 20, device="cuda")
    with pytest.raises(ValueError, match="training 0.50 GB"):
        E.HeldOut(["in_test"], d, cfg, reserved_bytes=500_000_000, total_memory=600_000_000, device="cuda")
    with open(tmp_path / "data" / "out_test_samples_128.json", "w") as f:
        json.dump([["p999_000", 0]], f)
    with pytest.raises(ValueError, match="not in the pickle"):
        E.HeldOut(["in_test", "out_test"], d, cfg, total_memory=1 << 40, device="cuda")
    with open(tmp_path / "data" / "in_test.pkl", "wb") as f:
        pickle.dump({"p1_000": np.zeros((200, 40), np.float32)}, f)
    with pytest.raises(ValueError, match="c_in"):
        E.HeldOut(["in_test"], d, cfg, total_memory=1 << 40, device="cuda")
    with pytest.raises(FileNotFoundError):
        E.HeldOut(["nope"], d, cfg, total_memory=1 << 40, device="cuda")
