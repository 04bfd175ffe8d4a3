"""CPU: the float64 YIN restatement (tests/_f0_ref.py) tracks known signals, its lag-choice semantics, the F0 metrics
of adaptive_voice_conversion_b200/f0.py against the restatement, the pair selection, evaluate.py's -f0 arguments and
avc_yin's argument checks (no launch: there is no GPU here)."""
import ctypes
import math
import os
import pickle
import random

import numpy as np
import pytest

import _f0_ref as R

SR, HOP, WIN = 24000, 300, 1024


def inner_frames(n, tau_max=480):
    """Frames whose span lies inside the signal (no reflection)."""
    half = (WIN + tau_max) // 2
    return [f for f in range(1 + n // HOP) if f * HOP - half >= 0 and f * HOP - half + WIN + tau_max <= n]


@pytest.mark.parametrize("f0", [55.0, 110.0, 180.0, 260.0, 450.0])
def test_restatement_tracks_harmonic_signals(f0):
    y = R.harmonic(f0, 0.5, phase_seed=int(f0))
    fr = inner_frames(len(y))
    out = R.yin(y, SR, HOP, frames=fr)
    f0h, voiced = R.voicing(out["tau"], out["aperiodicity"], out["energy"], SR)
    assert voiced.all()
    assert np.max(np.abs(f0h / f0 - 1)) < 5e-3


def test_restatement_tracks_a_glide():
    lo, hi, dur = 100.0, 300.0, 2.0
    y = R.harmonic(lambda t: lo + (hi - lo) * t / dur, dur)
    fr = inner_frames(len(y))
    out = R.yin(y, SR, HOP, frames=fr)
    f0h, voiced = R.voicing(out["tau"], out["aperiodicity"], out["energy"], SR)
    want = lo + (hi - lo) * np.asarray(fr) * HOP / SR / dur
    assert voiced.all()
    assert np.max(np.abs(f0h / want - 1)) < 2e-2


def test_noise_is_unvoiced_and_silence_is_unvoiced_and_finite():
    y = np.random.default_rng(0).standard_normal(SR).astype(np.float32) * 0.3
    out = R.yin(y, SR, HOP)
    _, voiced = R.voicing(out["tau"], out["aperiodicity"], out["energy"], SR)
    assert voiced.mean() <= 0.05
    z = np.zeros(SR // 2, np.float32)
    out = R.yin(z, SR, HOP)
    f0h, voiced = R.voicing(out["tau"], out["aperiodicity"], out["energy"], SR)
    assert not voiced.any()
    assert all(np.isfinite(out[k]).all() for k in ("tau", "aperiodicity", "energy"))
    assert (out["aperiodicity"] == 1.0).all() and (out["energy"] == 0).all()


def test_cmnd_of_zero_sums_is_one():
    d = np.array([0.0, 0.0, 0.0, 2.0, 1.0])
    np.testing.assert_array_equal(R.cmnd(d), [1.0, 1.0, 1.0, 3.0, 4.0 / 3.0])


def curve(vals):
    return np.asarray([1.0] + list(vals), np.float64)     # dp[0] unused


def test_choice_threshold_descent_tie_and_clamp():
    # the first tau below theta (5), then descent to the local minimum (7)
    dp = curve([1, 1, 1, 1, 0.09, 0.08, 0.05, 0.07, 0.01, 1])
    ts, delta = R.choose(dp, 2, 10, 0.1)
    assert ts == 7
    a, b, c = 0.08, 0.05, 0.07
    assert delta == pytest.approx((a - c) / (2 * (a - 2 * b + c)))
    # descent stops at tau_max
    dp = curve([1, 0.09, 0.08, 0.07, 0.06])
    assert R.choose(dp, 2, 5, 0.1) == (5, 0.0)
    # nothing below theta: argmin, the smallest tau on ties
    dp = curve([0.9, 0.5, 0.7, 0.5, 0.8])
    assert R.choose(dp, 1, 5, 0.1)[0] == 2
    # tau_min excludes earlier lags
    dp = curve([0.01, 0.5, 0.7, 0.4, 0.8, 0.9])
    assert R.choose(dp, 2, 6, 0.1)[0] == 4
    # a tie below theta: the descent stops at the first of equal values
    dp = curve([1, 0.05, 0.05, 0.2])
    assert R.choose(dp, 1, 4, 0.1)[0] == 2


def test_refinement_denominator_and_clamp():
    # tau* is the argmin over [3, 5] but d'(2) lies below it: a - 2b + c = -0.2 <= 0, no refinement
    dp = curve([0.9, 0.2, 0.5, 0.6, 0.7])
    assert R.choose(dp, 3, 5, 0.1) == (3, 0.0)
    # a vertex more than half a lag away is clamped: (0.45 - 0.9) / (2 * 0.35) = -0.64 -> -1/2
    dp = curve([0.9, 0.45, 0.5, 0.9, 0.95])
    assert R.choose(dp, 3, 5, 0.1) == (3, -0.5)
    # tau* = tau_max or tau* - 1 = 0: no refinement
    assert R.choose(curve([0.9, 0.5, 0.3]), 2, 3, 0.1) == (3, 0.0)
    assert R.choose(curve([0.05, 0.5, 0.3]), 1, 3, 0.1) == (1, 0.0)


def test_package_choice_matches_the_restatement_on_random_curves():
    """pair_scores, profile and voicing of the package equal the restatement on random curves and tracks."""
    from adaptive_voice_conversion_b200 import f0 as F
    rng = np.random.default_rng(1)
    for _ in range(50):
        n = int(rng.integers(2, 60))
        tau = rng.uniform(48, 480, n)
        ap = rng.uniform(0, 0.3, n)
        en = rng.uniform(0, 1, n) ** 6
        en[rng.random(n) < 0.1] = 0.0
        a = F.voicing(tau, ap, en, SR)
        b = R.voicing(tau, ap, en, SR)
        np.testing.assert_array_equal(a[1], b[1])
        np.testing.assert_array_equal(a[0], b[0])


def track(f0s, voiced):
    return np.asarray(f0s, np.float64), np.asarray(voiced, bool)


def test_pair_metrics_and_every_unvoiced_case():
    from adaptive_voice_conversion_b200 import f0 as F
    conv = track([100, 110, 121, 0, 140], [1, 1, 1, 0, 1])
    src = track([200, 210, 230, 240, 0], [1, 1, 1, 1, 0])
    tm, sm = math.log2(105), math.log2(220)
    got = F.pair_scores(conv, src, tm, sm)
    want = R.pair(conv, src, tm, sm)
    assert got == pytest.approx(want, rel=1e-14, abs=0)
    assert got[0] == 3 / 5
    mc = (math.log2(100) + math.log2(110) + math.log2(121) + math.log2(140)) / 4
    assert got[2] == pytest.approx(12 * abs(mc - tm)) and got[4] == 1.0
    # fewer than two frames voiced in both
    assert F.pair_scores(track([100, 110], [1, 0]), track([100, 110], [1, 1]), tm, sm) is None
    assert F.pair_scores(track([100, 110], [1, 1]), track([100, 110], [0, 1]), tm, sm) is None
    # a constant series over the common frames
    assert F.pair_scores(track([100, 100, 90], [1, 1, 0]), track([100, 120, 90], [1, 1, 1]), tm, sm) is None
    assert F.pair_scores(track([100, 120, 90], [1, 1, 0]), track([130, 130, 90], [1, 1, 1]), tm, sm) is None
    # a profile without a voiced frame
    assert F.pair_scores(conv, src, None, sm) is None and F.pair_scores(conv, src, tm, None) is None
    for case in [((track([100, 110], [1, 0]), track([100, 110], [1, 1])), (tm, sm)),
                 ((track([100, 100, 90], [1, 1, 0]), track([100, 120, 90], [1, 1, 1])), (tm, sm)),
                 ((conv, src), (None, sm))]:
        assert R.pair(*case[0], *case[1]) is None


def test_profiles_match_the_restatement():
    from adaptive_voice_conversion_b200 import f0 as F
    rng = np.random.default_rng(2)
    series = [np.log2(rng.uniform(80, 300, int(rng.integers(0, 40)))) for _ in range(6)]
    m, s, n = F.profile(series)
    rm, rs = R.profile(series)
    assert (m, s) == (rm, rs) and n == sum(len(x) for x in series)     # the same sequential sums
    assert F.profile([np.zeros(0)]) == (None, None, 0)


def test_measure_restatement_counts_unvoiced_pairs():
    rng = np.random.default_rng(3)
    real = {}
    for s in ("p1", "p2", "p3"):
        for i in range(3):
            T = int(rng.integers(20, 40))
            v = rng.random(T) < 0.7
            if s == "p3":
                v[:] = False                     # a speaker without a voiced frame
            real[f"{s}_{i:03d}"] = (np.where(v, rng.uniform(90, 250, T), np.nan), v)
    pairs = [("p1_000", ["p2_001"]), ("p2_000", ["p1_002"]), ("p1_001", ["p3_000"])]
    conv = [(np.where(real[u][1], real[u][0] * 1.1, np.nan), real[u][1].copy()) for u, _ in pairs]
    rows, n_unv, total, spk, prof = R.measure(pairs, real, conv)
    assert n_unv == 1 and sorted(rows) == [0, 1] and total["n"] == 2
    assert prof["p3"]["voiced"] == 0 and prof["p3"]["log2_mean"] is None
    assert set(spk) == {"p2", "p1"}


def test_pair_selection_is_the_speaker_measure_pairs():
    from adaptive_voice_conversion_b200 import f0 as F
    from adaptive_voice_conversion_b200.config import default_config
    from adaptive_voice_conversion_b200.mcd import min_frames
    from adaptive_voice_conversion_b200.speaker_eval import conversion_pairs, fewshot_pairs
    cfg = default_config(80)
    rng = random.Random(4)
    lengths = {f"p{300 + s}_{u:03d}": rng.choice([5, 12, 16, 17, 40, 300]) for s in range(6) for u in range(rng.randint(1, 6))}
    min_src, min_ref = min_frames(cfg)
    ms = max(min_src, min_ref)
    for seed, max_pairs in [(0, 0), (3, 4), (7, 0)]:
        utts, pairs, refs, res = F.select_pairs(cfg, lengths, seed, max_pairs)
        want, n_short = conversion_pairs(list(lengths), lengths, seed, max_pairs, ms, min_ref, ms)
        assert pairs == want and res["n_short"] == n_short and refs == [[r] for _, r in want]
        assert utts == sorted(u for u in lengths if lengths[u] >= ms)
        utts, pairs, refs, res = F.select_pairs(cfg, lengths, seed, max_pairs, n_refs=2)
        few, n_few = fewshot_pairs(want, list(lengths), lengths, 2, seed, min_ref, ms)
        assert pairs == few and refs == [r for _, r in few] and res["n_few"] == n_few and res["n_refs"] == 2


def test_f0_params():
    from adaptive_voice_conversion_b200.f0 import F0Params
    p = F0Params()
    assert (p.tau_min(SR), p.tau_max(SR)) == (48, 480) == R.taus(SR)
    assert p.min_samples(SR) == (1024 + 480) // 2 + 1
    assert p.theta() == float(np.float32(0.1)) != 0.1


def run_cli(argv):
    import importlib.util
    from conftest import ROOT
    spec = importlib.util.spec_from_file_location("evaluate_cli", os.path.join(ROOT, "evaluate.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.main(argv)


def test_cli_f0_arguments(tmp_path, capsys):
    base = ["-m", str(tmp_path / "none.ckpt"), "-d", str(tmp_path)]
    with pytest.raises(SystemExit):
        run_cli(base + ["-f0"])                                    # no attr.pkl
    assert "-f0 needs the mel statistics" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        run_cli(base + ["-f0", "-attr", str(tmp_path / "missing.pkl")])
    assert "missing.pkl does not exist" in capsys.readouterr().err
    with open(tmp_path / "attr.pkl", "wb") as f:
        pickle.dump({"mean": np.zeros(80), "std": np.ones(80)}, f)
    for bad, msg in [(["-gl_iters", "-1"], "-gl_iters"), (["-gl_momentum", "1.0"], "-gl_momentum"),
                     (["-gl_init", "random"], "invalid choice")]:
        with pytest.raises(SystemExit):
            run_cli(base + ["-f0"] + bad)
        assert msg in capsys.readouterr().err


def test_avc_yin_checks_every_argument_before_a_launch():
    from adaptive_voice_conversion_b200 import _lib as L
    lib = L.load()
    n0 = L.launch_count()
    def desc(**kw):
        d = L.AudioDesc(hop=300, n_seg=1, n_frames=10, n_samples=3000)
        d.segs, d.y = 16, 16
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    def call(d=None, win=1024, tmin=48, tmax=480, th=0.1, out=(16, 16, 16)):
        return lib.avc_yin(None if d is None else ctypes.byref(d), win, tmin, tmax, ctypes.c_float(th), *out, None)
    cases = [
        (lambda: call(None), L.ERR_INVALID, "null descriptor"),
        (lambda: call(desc(segs=None)), L.ERR_INVALID, "utterance table"),
        (lambda: call(desc(n_seg=0)), L.ERR_INVALID, "utterance table"),
        (lambda: call(desc(y=None)), L.ERR_INVALID, "null signal"),
        (lambda: call(desc(hop=0)), L.ERR_INVALID, "hop"),
        (lambda: call(desc(), out=(16, None, 16)), L.ERR_INVALID, "aperiodicity"),
        (lambda: call(desc(), tmin=0), L.ERR_INVALID, "tau_min"),
        (lambda: call(desc(), tmin=480, tmax=480), L.ERR_INVALID, "tau_min"),
        (lambda: call(desc(), win=479), L.ERR_INVALID, "win must be >= tau_max"),
        (lambda: call(desc(), win=L.YIN_MAX_SPAN - 479), L.ERR_UNSUPPORTED, "AVC_YIN_MAX_SPAN"),
        (lambda: call(desc(), th=0.0), L.ERR_INVALID, "threshold"),
        (lambda: call(desc(), th=1.5), L.ERR_INVALID, "threshold"),
        (lambda: call(desc(), th=float("nan")), L.ERR_INVALID, "threshold"),
        (lambda: call(desc(), th=float("inf")), L.ERR_INVALID, "threshold"),
    ]
    for fn, want, msg in cases:
        rc = fn()
        assert rc == want, (msg, rc)
        assert msg in L.last_error(), (msg, L.last_error())
    # zero frames: nothing to launch, and nothing is
    assert call(desc(n_frames=0), win=L.YIN_MAX_SPAN - 480, th=1.0) == L.OK
    assert L.launch_count() == n0


def test_header_constant_matches_the_binding():
    import subprocess
    import tempfile
    from adaptive_voice_conversion_b200 import _lib as L
    from conftest import ROOT
    prog = '#include <stdio.h>\n#include "avc_b200.h"\nint main(){printf("%d\\n", AVC_YIN_MAX_SPAN);return 0;}\n'
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "s.c")
        open(c, "w").write(prog)
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", os.path.join(td, "s")])
        assert int(subprocess.check_output([os.path.join(td, "s")])) == L.YIN_MAX_SPAN
