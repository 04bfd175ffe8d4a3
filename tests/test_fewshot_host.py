"""CPU: the host side of few-shot conversion (a speaker code pooled over several references of the target speaker).

* the -pairs target field: one file when it names an existing file (commas included), otherwise a comma-separated
  reference set whose every member must exist; the default output name; lines naming one set share one list object;
* the evaluators' extra reference draws against a literal restatement, and n_refs = 1 giving conversion_pairs' and
  parallel_triplets' pairs;
* AE.get_speaker_embeddings(groups=) validation errors raised before any launch;
* embed_speakers' set packing: every set whole in one batch of at most PADDED_BATCH_MAX references;
* the new kernels keep everything in registers (no stack, no spills), as tests/test_spk_resources.py checks for spk.cu.
"""
import os
import random
import re
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def cli():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import inference
    return inference


# ----------------------------------------------------------------------------- the -pairs target field
def test_pairs_target_field(tmp_path):
    inf = cli()
    for n in ("a", "b", "c", "d,e"):
        np.save(tmp_path / f"{n}.npy", np.zeros((40, 80), np.float32))
    a, b, c, de = (str(tmp_path / f"{n}.npy") for n in ("a", "b", "c", "d,e"))
    f = tmp_path / "pairs.txt"
    f.write_text(f"{a} {b}\n{a} {b},{c}\n{c} {de}\n{b} {b},{c} x.npy\n{a} {c},{a},{b}\n")
    pairs = inf.read_pairs(str(f))
    assert pairs == [(1, a, b, "a_to_b.wav"), (2, a, (b, c), "a_to_b.wav"), (3, c, de, "c_to_d,e.wav"),
                     (4, b, (b, c), "x.npy"), (5, a, (c, a, b), "a_to_c.wav")]
    # a missing member of a set, and a comma list whose parts do not exist, name the line
    for text, msg in ((f"{a} {b},{tmp_path / 'missing.npy'}\n", "line 1.*missing.npy"),
                      (f"{a} {a}\n{a} {tmp_path / 'd'},{tmp_path / 'e.npy'}\n", "line 2"),
                      (f"{a} {b},\n", "line 1")):
        g = tmp_path / "bad.txt"
        g.write_text(text)
        with pytest.raises(ValueError, match=msg):
            inf.read_pairs(str(g))
    # frames of every member are checked, naming the line and the member
    with pytest.raises(ValueError, match=f"line 2: target {re.escape(c)} has 8 frames"):
        inf.check_frames([(2, a, (b, c), "o.npy")], [40], [[40, 8]], (17, 9))
    inf.check_frames([(2, a, (b, c), "o.npy")], [40], [[40, 9]], (17, 9))


def test_pairs_share_one_set_object(tmp_path):
    """convert_pairs: single-target lines in one inference_padded call (today's), set lines in another, lines naming
    the same set with one list object (so inference_padded embeds it once)."""
    inf = cli()
    calls = []

    class Fake:
        def inference_padded(self, xs, x_conds):
            calls.append((list(xs), list(x_conds)))
            return [f"dec{len(calls)}_{i}" for i in range(len(xs))]

    mels = {p: torch.zeros(1) + i for i, p in enumerate(("s1", "s2", "t1", "t2", "t3"))}
    pairs = [(1, "s1", ("t1", "t2"), "o1"), (2, "s2", "t3", "o2"), (3, "s2", ("t1", "t2"), "o3"),
             (4, "s1", ("t2", "t1"), "o4"), (5, "s1", "t1", "o5")]
    decs = inf.convert_pairs(Fake(), pairs, mels)
    assert decs == ["dec2_0", "dec1_0", "dec2_1", "dec2_2", "dec1_1"]
    (xs1, c1), (xs2, c2) = calls
    assert [x is mels[s] for x, s in zip(xs1, ("s2", "s1"))] == [True, True] and c1 == [mels["t3"], mels["t1"]]
    assert c2[0] is c2[1] and c2[0] is not c2[2]
    assert [[t is mels[n] for t, n in zip(s, names)] for s, names in zip(c2, (("t1", "t2"),) * 2 + (("t2", "t1"),))] == \
        [[True, True]] * 3


# ----------------------------------------------------------------------------- the evaluators' draws
def _set(n_spk=5, per=(1, 2, 3, 5, 8), seed=0):
    g = random.Random(seed)
    utts, lengths = [], {}
    for s in range(n_spk):
        for k in range(per[s % len(per)]):
            u = f"p{300 + s}_{k:03d}.wav"
            utts.append(u)
            lengths[u] = g.choice([5, 12, 40, 200])
    return utts, lengths


def restate_spk(pairs, utts, lengths, K, seed, min_ref, min_set):
    rng2 = random.Random(seed + 1)
    out, n_few = [], 0
    for u, r in pairs:
        spk = r.split("_")[0]
        cand = sorted(v for v in utts if v.split("_")[0] == spk and v != r and lengths[v] >= min_ref)
        if 1 + len(cand) < K:
            n_few += 1
            continue
        refs = [r] + rng2.sample(cand, K - 1)
        left = [v for v in utts if v.split("_")[0] == spk and v not in refs and lengths[v] >= min_set]
        if not left:
            n_few += 1
            continue
        out.append((u, refs))
    return out, n_few


@pytest.mark.parametrize("K", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("seed", [0, 7])
def test_spk_fewshot_draws(K, seed):
    from adaptive_voice_conversion_b200.speaker_eval import conversion_pairs, fewshot_pairs
    utts, lengths = _set(6, seed=seed)
    for max_pairs in (0, 3):
        pairs, _ = conversion_pairs(utts, lengths, seed, max_pairs, 17, 9, 17)
        got = fewshot_pairs(pairs, utts, lengths, K, seed, 9, 17)
        assert got == restate_spk(pairs, utts, lengths, K, seed, 9, 17)
        if K == 1:
            assert got == ([(u, [r]) for u, r in pairs], 0)
        else:
            # the first references are exactly n_refs = 1's, less the dropped pairs
            kept = [(u, refs[0]) for u, refs in got[0]]
            assert kept == [p for p in pairs if p in kept] and len(kept) + got[1] == len(pairs)
            assert all(len(set(refs)) == K for _, refs in got[0])


def restate_mcd(trip, utts, texts, lengths, K, seed, min_ref):
    rng2 = random.Random(seed + 1)
    out, n_few = [], 0
    for s, r, g in trip:
        spk = g.split("_")[0]
        cand = sorted(v for v in utts if v.split("_")[0] == spk and v != r and texts.get(v) != texts[g]
                      and lengths[v] >= min_ref)
        if 1 + len(cand) < K:
            n_few += 1
            continue
        out.append((s, [r] + rng2.sample(cand, K - 1), g))
    return out, n_few


@pytest.mark.parametrize("K", [1, 2, 3, 5])
def test_mcd_fewshot_draws(K):
    from adaptive_voice_conversion_b200.mcd import fewshot_triplets, parallel_triplets
    utts, lengths = _set(5, per=(3, 4, 6, 2, 8), seed=3)
    g = random.Random(1)
    texts = {u: g.choice(["one", "two", "three"]) for u in utts if g.random() < 0.9}
    for max_pairs in (0, 4):
        trip, _ = parallel_triplets(utts, texts, lengths, 0, max_pairs, 17, 9)
        got = fewshot_triplets(trip, utts, texts, lengths, K, 0, 9)
        assert got == restate_mcd(trip, utts, texts, lengths, K, 0, 9)
        if K == 1:
            assert got == ([(s, [r], t) for s, r, t in trip], 0)
        for s, refs, t in got[0]:
            assert all(texts.get(r) != texts[t] for r in refs) and len(set(refs)) == K


# ----------------------------------------------------------------------------- groups validation
def test_groups_rejected_before_any_launch():
    from adaptive_voice_conversion_b200 import _lib as L
    from adaptive_voice_conversion_b200.model import _check_groups
    L.load()
    x = torch.zeros(5, 80, 100)
    n0 = L.launch_count()
    assert _check_groups(torch.tensor([0, 2, 3, 5]), x, "g").tolist() == [0, 2, 3, 5]
    assert _check_groups(torch.tensor([0, 5], dtype=torch.int16), x, "g").dtype == torch.int32
    bad = [torch.tensor([1, 3, 5]),              # not starting at 0
           torch.tensor([0, 3, 4]),              # not ending at B
           torch.tensor([0, 3, 3, 5]),           # an empty group
           torch.tensor([0, 4, 3, 5]),           # decreasing
           torch.tensor([0]),                    # no group
           torch.tensor([0, 1, 2, 3, 4, 5, 5]),  # more groups than rows
           torch.tensor([[0, 5]]),               # wrong shape
           torch.tensor([0.0, 5.0]),             # wrong dtype
           torch.tensor([False, True]),
           [0, 5]]                               # not a tensor
    for v in bad:
        with pytest.raises(L.AvcError):
            _check_groups(v, x, "g")
    assert L.launch_count() == n0


def test_engine_groups_need_lengths_and_inference():
    from adaptive_voice_conversion_b200 import _lib as L
    from adaptive_voice_conversion_b200.engine import Engine, Lengths
    e = Engine.__new__(Engine)           # the check comes before any use of the engine's state
    with pytest.raises(L.AvcError, match="groups"):
        e.speaker_fwd({}, torch.zeros(2, 80, 64), False, groups=torch.tensor([0, 2]))
    with pytest.raises(L.AvcError, match="groups"):
        e.speaker_fwd({}, torch.zeros(2, 80, 64), True, lens=Lengths(torch.tensor([64, 64])), groups=torch.tensor([0, 2]))


# ----------------------------------------------------------------------------- set packing
@pytest.mark.parametrize("seed", range(5))
def test_pack_sets(seed):
    from adaptive_voice_conversion_b200.inference import PADDED_BATCH_MAX, pack_sets, padded_extent
    g = random.Random(seed)
    n = g.choice([1, 5, 64, 300])
    sizes = [g.choice([1, 1, 4, 16, 63, 64]) for _ in range(n)]
    lens = [g.randint(9, 1500) for _ in range(n)]
    batches = pack_sets(sizes, lens)
    seen = sorted(i for idx, _ in batches for i in idx)
    assert seen == list(range(n))                                     # every set once, whole
    order = [i for idx, _ in batches for i in idx]
    assert order == sorted(range(n), key=lambda i: (lens[i], i))
    for k, (idx, T) in enumerate(batches):
        assert sum(sizes[i] for i in idx) <= PADDED_BATCH_MAX
        assert T == padded_extent(max(lens[i] for i in idx)) and T >= max(lens[i] for i in idx)
        if k + 1 < len(batches):                                      # greedy: the next set did not fit
            assert sum(sizes[i] for i in idx) + sizes[batches[k + 1][0][0]] > PADDED_BATCH_MAX
    with pytest.raises(ValueError, match="set 1"):
        pack_sets([3, 65], [10, 10])
    with pytest.raises(ValueError, match="set 0"):
        pack_sets([0], [10])


def test_embed_speakers_rejects_bad_sets():
    from adaptive_voice_conversion_b200 import _lib as L
    from adaptive_voice_conversion_b200.config import default_config
    from adaptive_voice_conversion_b200.inference import Inferencer
    inf = Inferencer.__new__(Inferencer)
    inf.config = default_config(80)
    n0 = L.launch_count()
    with pytest.raises(ValueError, match="set 1 has 65 references"):
        inf.embed_speakers([[torch.zeros(20, 80)], [torch.zeros(20, 80)] * 65])
    with pytest.raises(ValueError, match="reference 2 of set 0 has 8 frames"):
        inf.embed_speakers([[torch.zeros(20, 80), torch.zeros(9, 80), torch.zeros(8, 80)]])
    with pytest.raises(ValueError, match="set 0 must be a non-empty list"):
        inf.embed_speakers([[]])
    with pytest.raises(ValueError, match="mixes"):
        inf.inference_padded([torch.zeros(20, 80)] * 2, [torch.zeros(20, 80), [torch.zeros(20, 80)]])
    assert L.launch_count() == n0


# ----------------------------------------------------------------------------- kernel resources
KERNELS = ("time_mean_grouped_kernel", "time_mean_fwd_kernel", "spk_group_mean_kernel")


def test_fewshot_kernels_have_no_stack_and_no_spills():
    from adaptive_voice_conversion_b200 import _lib as L
    L.load()
    out = subprocess.run(["cuobjdump", "-res-usage", L.LIB_PATH], capture_output=True, text=True).stdout
    res, fn = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            fn = m.group(1)
        elif fn and any(k in fn for k in KERNELS) and "REG:" in line:
            res[fn] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
    assert sorted(k for k in KERNELS if any(k in fn for fn in res)) == sorted(KERNELS), sorted(res)
    for fn, r in res.items():
        assert r["STACK"] == 0 and r["LOCAL"] == 0, (fn, r)
