"""CPU: the float64 restatement of the pitch shift (tests/_pshift_ref.py) against an FFT cepstrum and on spectra whose
shift is known (identity, a pure envelope, a comb of peaks, the held edge); the shift arithmetic of match mode; the
-pitch_shift arguments of inference.py and evaluate.py; and the C ABI's argument checks."""
import importlib.util
import os
import types

import numpy as np
import pytest

import _pshift_ref as R
from conftest import ROOT

NB = 1025


def smooth_ell(Q, seed=0):
    """A log spectrum holding only quefrencies below Q."""
    rng = np.random.default_rng(seed)
    c = rng.standard_normal(Q) / (1.0 + np.arange(Q))
    return c @ R.cos_matrix(Q, NB)


def test_cepstrum_is_the_dct_of_the_even_extension():
    ell = np.random.default_rng(1).standard_normal((3, NB))
    ext = np.concatenate([ell, ell[:, -2:0:-1]], axis=1)          # the even extension, period N = 2048
    want = np.fft.rfft(ext, axis=1).real / ext.shape[1]
    for Q in (1, 40, 1024):
        assert np.allclose(R.cepstrum(ell, Q), want[:, :Q], rtol=0, atol=1e-12)


def test_ratio_one_is_the_identity():
    S = np.exp(np.random.default_rng(2).standard_normal((4, NB)))
    S[0, :10] = 0.0
    assert np.array_equal(R.pitch_shift(S, 1.0), S)


@pytest.mark.parametrize("ratio", [0.25, 0.8, 1.5, 4.0])
def test_a_pure_envelope_is_unchanged(ratio):
    Q = 40
    S = np.exp(smooth_ell(Q - 1) - 2.0)
    assert np.all(S > 1e-4)
    ell, E, F = R.split(S, Q)
    assert np.max(np.abs(F)) < 1e-10
    assert np.allclose(R.pitch_shift(S, ratio, Q), S, rtol=1e-9, atol=0)


def comb(delta, width=1.2, env=None):
    k = np.arange(NB)
    ell = np.log(1e-3 + sum(np.exp(-0.5 * ((k - j * delta) / width) ** 2) for j in range(1, NB // delta + 1)))
    return np.exp(ell + (0.0 if env is None else env))


def peaks(x, lo=5, hi=None):
    """Local maxima more than e^3 above the median (the lifter's ripple between the comb's peaks stays below)."""
    i = np.flatnonzero((x[1:-1] > x[:-2]) & (x[1:-1] >= x[2:]) & (x[1:-1] > np.exp(3.0) * np.median(x))) + 1
    return i[(i >= lo) & (i < (hi or len(x) - 5))]


@pytest.mark.parametrize("delta,ratio", [(20, 1.25), (24, 0.75), (16, 2.0 ** (7 / 12))])
def test_a_comb_of_peaks_spaced_delta_comes_out_spaced_alpha_delta(delta, ratio):
    env = 0.5 * smooth_ell(8, seed=3)
    S = comb(delta, env=env)
    out = R.pitch_shift(S, ratio)[0]
    top = min(NB - 1, (NB - 1) * ratio) - 2 * delta * ratio
    got = peaks(out, lo=int(delta * ratio / 2), hi=int(top))
    want = np.arange(1, 200) * delta * ratio
    want = want[(want >= delta * ratio / 2) & (want < top)]
    assert len(got) == len(want)
    assert np.max(np.abs(got - want)) <= 1.0
    # the envelope is kept: the shifted peaks' heights follow exp(env) at their new bins, not their old ones
    h = np.log(out[got])
    assert np.corrcoef(h, env[got])[0, 1] > 0.9


def test_the_edge_is_held_for_ratios_below_one():
    S = comb(20, env=0.5 * smooth_ell(8, seed=4))
    for ratio in (0.5, 0.8):
        ell, E, F = R.split(S, 40)
        out = R.pitch_shift(S, ratio)[0]
        held = np.arange(NB) / np.float32(ratio) >= NB - 1
        assert held.sum() >= NB * (1 - ratio) - 2
        assert np.allclose(np.log(out[held]), E[0, held] + F[0, -1], rtol=0, atol=1e-12)


def test_invalid_ratios_give_nan():
    S = np.ones((1, NB))
    for a in (0.0, -1.0, np.inf, np.nan):
        assert np.isnan(R.pitch_shift(S, a)).all()


# ----------------------------------------------------------------------------- match arithmetic
def trk(f0s):
    f = np.asarray(f0s, np.float64)
    return np.where(np.isnan(f), np.nan, f), ~np.isnan(f)


def test_match_arithmetic_on_hand_built_tracks():
    from adaptive_voice_conversion_b200.f0 import shifts_from_tracks
    nan = np.nan
    convs = [trk([150.0, nan, 150.0, 150.0]),            # matched: 12 log2(220/150)
             trk([100.0, 200.0]),                        # mean log2 is log2(100 * sqrt 2)
             trk([50.0, 50.0]),                          # 5 octaves below: clamped
             trk([nan, nan]),                            # no voiced conversion frame
             trk([150.0])]                               # no voiced reference frame
    refs = [[trk([220.0, nan]), trk([220.0, 220.0])],
            [trk([400.0])],
            [trk([1600.0])],
            [trk([200.0])],
            [trk([nan, nan]), trk([nan])]]
    shifts, info = shifts_from_tracks(convs, refs)
    assert shifts[0] == pytest.approx(12 * np.log2(220 / 150), abs=1e-12)
    assert shifts[1] == pytest.approx(12 * (np.log2(400) - np.log2(100 * np.sqrt(2))), abs=1e-12)
    assert shifts[2] == 24.0 and info[2]["clamped"] and not info[2]["unmatched"]
    assert shifts[3] == 0.0 and info[3]["unmatched"] and info[3]["voiced_conv"] == 0
    assert shifts[4] == 0.0 and info[4]["unmatched"] and info[4]["voiced_refs"] == 0
    assert (info[0]["voiced_conv"], info[0]["voiced_refs"]) == (3, 3)
    assert not any(d["clamped"] or d["unmatched"] for d in info[:2])
    assert shifts_from_tracks([trk([1600.0])], [[trk([50.0])]])[0] == [-24.0]


def test_semitone_checks():
    from adaptive_voice_conversion_b200.vocoder import _semitones
    assert _semitones(3, 2, "x") == [3.0, 3.0]
    assert _semitones([-24, 24], 2, "x") == [-24.0, 24.0]
    for bad in (24.01, -30, float("nan"), float("inf")):
        with pytest.raises(ValueError, match="pitch shift"):
            _semitones(bad, 1, "x")
    with pytest.raises(ValueError, match="2 shifts for 3"):
        _semitones([0, 1], 3, "x")


# ----------------------------------------------------------------------------- command lines
def load_script(name):
    spec = importlib.util.spec_from_file_location(f"{name}_cli", os.path.join(ROOT, f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_inference_pitch_shift_arguments(capsys):
    inf = load_script("inference")

    def check(argv):
        p = inf.parser()
        args = p.parse_args(argv)
        inf.check_args(p, args)
        return args
    one = ["-s", "a.wav", "-t", "b.wav", "-o", "o.wav"]
    assert check(one).semitones == 0.0
    assert check(one + ["-pitch_shift", "-24"]).semitones == -24.0
    assert check(one + ["-pitch_shift", "match"]).semitones == "match"
    assert check(["-s", "a.wav", "-t", "b.wav", "c.wav", "-o", "o.wav", "-pitch_shift", "match"]).semitones == "match"
    assert check(["-s", "a.wav", "-t", "b.wav", "-o", "o.npy"]).semitones == 0.0
    assert check(["-pairs", "p.txt", "-o", "d", "-pitch_shift", "3.5"]).semitones == 3.5
    assert check(["-pairs", "p.txt", "-o", "d", "-pitch_shift", "match"]).semitones == "match"
    assert check(["-s", "a.wav", "-bank", "b.pt", "-speaker", "p1", "-o", "o.wav", "-pitch_shift", "2"]).semitones == 2
    assert check(["-s", "a.wav", "-bank", "b.pt", "-morph", "p1@0", "-o", "o.wav", "-pitch_shift", "-2"]).semitones == -2
    for argv, msg in [
        (one + ["-pitch_shift", "24.5"], "[-24, 24]"),
        (one + ["-pitch_shift", "-25"], "[-24, 24]"),
        (one + ["-pitch_shift", "nan"], "finite"),
        (one + ["-pitch_shift", "inf"], "finite"),
        (one + ["-pitch_shift", "up"], "a number of semitones or 'match'"),
        (["-s", "a.wav", "-t", "b.wav", "-o", "o.npy", "-pitch_shift", "2"], ".npy output"),
        (["-s", "a.wav", "-t", "b.wav", "-o", "o.npy", "-pitch_shift", "match"], ".npy output"),
        (["-s", "a.wav", "-bank", "b.pt", "-speaker", "p1", "-o", "o.wav", "-pitch_shift", "match"], "banked"),
        (["-s", "a.wav", "-bank", "b.pt", "-morph", "p1@0", "-o", "o.wav", "-pitch_shift", "match"], "banked"),
    ]:
        with pytest.raises(SystemExit):
            check(argv)
        assert msg in capsys.readouterr().err, argv


def test_pairs_match_refuses_a_bank_line_before_the_gpu(tmp_path):
    inf = load_script("inference")
    for name in ("a.wav", "b.wav"):
        (tmp_path / name).write_bytes(b"")
    pf = tmp_path / "pairs.txt"
    pf.write_text(f"# header\n{tmp_path / 'a.wav'} {tmp_path / 'b.wav'}\n\n{tmp_path / 'b.wav'} @p225:0.5,p226:0.5\n")
    args = types.SimpleNamespace(pairs=str(pf), bank="bank.pt", semitones="match", output=str(tmp_path / "out"))
    with pytest.raises(ValueError, match=r"pairs.txt line 4: .*@p225:0.5,p226:0.5"):
        inf.run_pairs(args, {})
    assert not (tmp_path / "out").exists()


def test_evaluate_pitch_shift_arguments(tmp_path, capsys):
    ev = load_script("evaluate")
    base = ["-m", str(tmp_path / "none.ckpt"), "-d", str(tmp_path)]
    with pytest.raises(SystemExit):
        ev.main(base + ["-pitch_shift", "match"])
    assert "-pitch_shift needs -f0" in capsys.readouterr().err
    with pytest.raises(SystemExit):
        ev.main(base + ["-f0", "-pitch_shift", "3"])
    assert "invalid choice" in capsys.readouterr().err


def test_avc_pitch_shift_checks_every_argument_before_a_launch():
    from adaptive_voice_conversion_b200 import _lib as L
    lib = L.load()
    n0 = L.launch_count()
    A, B = 1 << 20, 1 << 30                                   # far apart: no overlap for these row counts

    def call(mag=A, ratio=16, out=B, rows=8, n_bins=1025, lifter=40):
        return lib.avc_pitch_shift(mag, ratio, out, rows, n_bins, lifter, None)
    cases = [
        (lambda: call(mag=None), L.ERR_INVALID, "null"),
        (lambda: call(ratio=None), L.ERR_INVALID, "null"),
        (lambda: call(out=None), L.ERR_INVALID, "null"),
        (lambda: call(rows=0), L.ERR_INVALID, "rows"),
        (lambda: call(lifter=0), L.ERR_INVALID, "lifter"),
        (lambda: call(lifter=1025), L.ERR_INVALID, "lifter"),
        (lambda: call(n_bins=513, lifter=40), L.ERR_UNSUPPORTED, "n_bins"),
        (lambda: call(n_bins=2049, lifter=1500), L.ERR_UNSUPPORTED, "n_bins"),
        (lambda: call(out=A), L.ERR_INVALID, "overlaps"),
        (lambda: call(out=A + 4 * 1025 * 8 - 4), L.ERR_INVALID, "overlaps"),
        (lambda: call(mag=B + 4, out=B), L.ERR_INVALID, "overlaps"),
    ]
    for fn, want, msg in cases:
        rc = fn()
        assert rc == want, (msg, rc)
        assert msg in L.last_error(), (msg, L.last_error())
    assert L.launch_count() == n0
