"""GPU: the streaming kernels avc_rtisi_la and avc_stft_window (csrc/audio.cu) called through the C ABI with tables
built here, so that every layout the ABI accepts is reachable, not only those streaming.Rtisi.prepare produces.

1. every RTISI-LA frame step, at every (win, hop) region the ABI accepts and look-ahead 0, 1, 3 and 7, matches the
   float64 restatement (tests/_rtisi_ref.py) run from the kernel's own float32 state, for K 0 to 32 iterations,
   de-emphasis 0, 0.97, 1 and -0.97, and magnitudes of a harmonic signal, random, all zero and a single bin;
2. a stream's frames split into launches of 0, 1, nb - 1, nb and 2 nb + 1 frames, with and without the close in the
   last one, give the bits of one frame per launch (nb = look-ahead + 1); this carries check 1 to multi-frame launches;
3. closes at T = 0, 1, T < nb and right after a commit give hop (T - 1) samples in all;
4. 1 024 streams in random phases on permuted slots give the bits each gets alone, and idle slots keep theirs;
5. every argument check gives its code and message before any launch;
6. translation invariance: a state (or an analysis entry) shifted by any number of frames gives the same bits, with
   positions past 2^31 and 2^32 samples (RTISI-LA, avc_stft_window and avc_yin_window), and at hop 1 up to 2^31 - 1
   frames;
7. avc_stft_window equals avc_stft bit for bit on ragged tables of entries at random origins.

Each launch's output sits between sentinel guards, with NaN gaps between the streams' ranges: the kernel writes
exactly the samples Rtisi.prepare's formula gives each stream, and nothing else.  The float64 bounds are about 3x the
worst error measured on the H100 (DESIGN.md section 6); each case prints its worst."""
import ctypes as C

import numpy as np
import pytest
import torch

import _rtisi_ref as R
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200.vocoder import _SEG, _ptr
from test_gpu_vocoder_kernels import GAP_NAN, PAIRS as STFT_PAIRS, Guarded, bits, signals, stft_lengths

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NFFT, NBIN = 2048, 1025
GAP_BITS = np.array([GAP_NAN], np.float32).view(np.uint32)[0]
STATE_NAN = np.array([0x7FC0D00D], np.uint32).view(np.float32)[0]   # idle slots' pattern

# every region of the ABI: even win <= 2048, 0 < hop <= win / 2
PAIRS = [(1200, 300), (2048, 1024), (2048, 512), (600, 150), (300, 150), (2046, 1023), (1200, 350), (2048, 7),
         (4, 2), (4, 1), (2, 1)]
LAS = [0, 1, 3, 7]
DEEMPHS = [0.0, 0.97, 1.0, -0.97]
KINDS = ["harmonic", "random", "zero", "single_bin"]

# |kernel - float64| / (peak |float64| of the step's output or of the buffered frames).  K <= 1: a step is one
# projection from the kernel's state.  K > 1: iterating amplifies the float32 rounding (see STEP_TOL in
# test_gpu_stream.py); the first step is left out when K > 1, as there.  About 3x the worst measured on 1x H100 80GB
# HBM3 (700 W power limit): K <= 1 1.8e-4 (a close at T = nb + 2, win 1200, hop 300), K > 1 1.44e-4 (random
# magnitudes at win 2048, hop 7, K 8).  What dominates is the phase S E/|E| at bins where |E| is small: float32 rounds
# E by about 2^-24 of the sum of its terms, and the phase moves by that over |E|.  Harmonic and single-bin magnitudes
# give 3e-8 to 2e-6 at K <= 1; random magnitudes, consistent with no signal, have many near-zero bins and give 8e-5.
TOL_ONE = 6e-4
TOL_ITER = 5e-4


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


# ------------------------------------------------------------------ RTISI-LA helpers
class Pool:
    """State slots of one (win, hop, look-ahead), as avc_rtisi_state_floats lays them out."""

    def __init__(self, win, hop, la, slots):
        self.win, self.hop, self.la, self.nb = win, hop, la, la + 1
        self.stride = int(L.load().avc_rtisi_state_floats(win, la))
        self.state = torch.zeros(slots, self.stride, device=DEV)
        self.count = torch.zeros(slots, 2, dtype=torch.int32, device=DEV)

    def snapshot(self, slot):
        return self.state[slot].clone(), self.count[slot].clone()

    def restore(self, slot, snap):
        self.state[slot].copy_(snap[0])
        self.count[slot].copy_(snap[1])

    def ref_state(self, slot):
        """The slot as the restatement's State (float64 copies of the kernel's float32 values)."""
        win, nb = self.win, self.nb
        s = self.state[slot].double().cpu().numpy()
        c, nbuf = (int(v) for v in self.count[slot].cpu())
        st = R.State(win, self.hop, self.la)
        st.c, st.nbuf, st.carry = c, nbuf, float(s[nb * win + nb * NBIN + win])
        st.num = s[nb * win + nb * NBIN:nb * win + nb * NBIN + win].copy()
        for F in range(c, c + nbuf):
            st.fr[F] = s[(F % nb) * win:(F % nb + 1) * win].copy()
            st.mag[F] = s[nb * win + (F % nb) * NBIN:nb * win + (F % nb + 1) * NBIN].copy()
        return st


def n_released(c, nbuf, p, close, win, hop, la):
    """Rtisi.prepare's formula: (samples released, counts after) for p new frames on counts (c, nbuf)."""
    rel = lambda k: max(0, k * hop - win // 2)   # noqa: E731
    if close:
        T = c + nbuf + p
        return max(0, (T - 1) * hop) - rel(c), (T, 0)
    nb2 = min(nbuf + p, la)
    c2 = c + nbuf + p - nb2
    return rel(c2) - rel(c), (c2, nb2)


def rtisi_desc(pool, K, deemph, n, mag, i32, out_off, y):
    return L.RtisiDesc(n_fft=NFFT, hop=pool.hop, win=pool.win, lookahead=pool.la, n_iter=K, n_streams=n,
                       deemph=deemph, mag=_ptr(mag), mag_off=_ptr(i32[:n + 1]), slot=_ptr(i32[n + 1:2 * n + 1]),
                       close=_ptr(i32[2 * n + 1:]), out_off=_ptr(out_off), y=_ptr(y), state=_ptr(pool.state),
                       count=_ptr(pool.count))


def launch(pool, K, deemph, entries, gap=11):
    """One avc_rtisi_la launch of entries [(slot, mags float32 [p, NBIN], close)].  Each stream's range of y lies
    between NaN gaps inside sentinel guards; asserts that the kernel wrote exactly Rtisi.prepare's count of samples
    for each stream and nothing else, and that the counts advanced as that formula says.  Returns the samples."""
    counts = pool.count.cpu().numpy()
    rows, offs, slots, closes, starts, ns, after = [], [0], [], [], [], [], []
    pos = gap
    for slot, m, close in entries:
        c, nbuf = (int(v) for v in counts[slot])
        n, cnt = n_released(c, nbuf, len(m), close, pool.win, pool.hop, pool.la)
        rows.append(np.asarray(m, np.float32).reshape(-1, NBIN))
        offs.append(offs[-1] + len(m))
        slots.append(slot)
        closes.append(int(close))
        starts.append(pos)
        ns.append(n)
        after.append(cnt)
        pos += n + gap
    y = Guarded(pos, np.full(pos, GAP_NAN, np.float32))
    mag = torch.from_numpy(np.concatenate(rows + [np.zeros((1, NBIN), np.float32)])).to(DEV)
    i32 = torch.tensor(offs + slots + closes, dtype=torch.int32, device=DEV)
    out_off = torch.tensor(starts, dtype=torch.int64, device=DEV)
    n = len(entries)
    L.check(L.load().avc_rtisi_la(C.byref(rtisi_desc(pool, K, deemph, n, mag, i32, out_off, y.t)), stream()),
            "avc_rtisi_la")
    torch.cuda.synchronize()
    y.check("avc_rtisi_la y")
    h = y.np()
    written = h.view(np.uint32) != GAP_BITS
    want = np.zeros(pos, bool)
    for s0, k in zip(starts, ns):
        want[s0:s0 + k] = True
    assert np.array_equal(written, want), ("released samples differ from Rtisi.prepare's count", ns,
                                           np.flatnonzero(written != want)[:8])
    got_counts = pool.count.cpu().numpy()
    for slot, cnt in zip(slots, after):
        assert tuple(int(v) for v in got_counts[slot]) == cnt, (slot, tuple(got_counts[slot]), cnt)
    return [h[s0:s0 + k].copy() for s0, k in zip(starts, ns)]


def harmonic_mags(win, hop, T, seed):
    """|STFT| at (win, hop) of R.harmonic, frames 0 .. T-1, as float32."""
    n = max(hop * (T - 1), 4 * NFFT)
    y = np.pad(R.harmonic(n, 24000, seed=seed), NFFT // 2, mode="reflect")
    w = np.zeros(NFFT)
    off = (NFFT - win) // 2
    w[off:off + win] = R.hann(win)
    return np.abs(np.stack([np.fft.rfft(y[f * hop:f * hop + NFFT] * w) for f in range(T)])).astype(np.float32)


def make_mags(kind, win, hop, T, rng):
    if kind == "harmonic":
        return harmonic_mags(win, hop, T, int(rng.integers(1 << 20)))
    if kind == "random":
        return rng.uniform(0.0, 2.0, (T, NBIN)).astype(np.float32)
    if kind == "zero":
        return np.zeros((T, NBIN), np.float32)
    m = np.zeros((T, NBIN), np.float32)          # one non-zero bin per row, at a row-dependent bin
    for f in range(T):
        m[f, int(rng.integers(0, NBIN))] = rng.uniform(0.5, 3.0)
    return m


def perturbed_step(st, mags, close, K, deemph, seed):
    """R.step with every projection's output moved by float32-sized rounding of the sums it is made of (2^-24 of
    sum |S| / 1024 per sample, seeded): how far float32 arithmetic alone can move the float64 result."""
    rng = np.random.default_rng(seed)
    orig = R.project

    def noisy(e, mag, win):
        out = orig(e, mag, win)
        return out + rng.standard_normal(len(out)) * 2.0 ** -24 * np.abs(mag).sum() / (NFFT // 2)
    R.project = noisy
    try:
        return R.step(st, mags, close, K, deemph)
    finally:
        R.project = orig


def step_errors(st, ref, got, after, pool, fr_peak):
    """(output error, frames error), each relative to its scale (see TOL_ONE); None where there is nothing to compare.
    An all-zero reference must be matched exactly."""
    eo = ef = None
    if len(ref):
        # the released samples are (numerator + frames) / window sum-square: scaled by the larger of their own peak
        # and the peak of the terms summed (a lone sample near a cancellation would otherwise set its own scale)
        pk = max(np.abs(ref).max(), fr_peak)
        if pk == 0:
            assert (got == 0).all(), "an all-zero stream gives exactly 0"
            eo = 0.0
        else:
            eo = float(np.abs(got - ref).max() / pk)
    if after is not None and st.nbuf:
        nb, win = pool.nb, pool.win
        pk = max(np.abs(v).max() for v in st.fr.values())
        e = max(np.abs(after[(F % nb) * win:(F % nb + 1) * win] - st.fr[F]).max() for F in range(st.c, st.c + st.nbuf))
        if pk == 0:
            assert e == 0
            ef = 0.0
        else:
            ef = float(e / pk)
    return eo, ef


def checked_step(pool, slot, mags, close, K, deemph, skip=False):
    """One launch of one stream, compared with R.step from the kernel's state before it.  Returns (the worst relative
    error, None when skipped; the samples released; True when the values were set aside as ill-conditioned).

    A step whose comparison exceeds the bound is set aside only when the float64 reference itself moves by more than
    the bound under float32-sized rounding of its projections (perturbed_step): the float32 result is then not
    determined to the bound by its inputs.  This happens at win 4: a frame that enters with phase 0 is the far tail of
    a pulse at sample 0 of n_fft, its four samples about 1e-9 of sum |S| / 1024, so its float32 value is rounding noise,
    and the next projection takes its phase from it.  Counts, totals and the sentinel checks still apply."""
    st = pool.ref_state(slot)
    st0 = st.copy()
    fr_peak = max([np.abs(v).max() for v in st.fr.values()] + [np.abs(st.num).max()])
    mags64, de = np.asarray(mags, np.float64), float(np.float32(deemph))
    ref = R.step(st, mags64, close, K, de)
    got = launch(pool, K, deemph, [(slot, mags, close)])[0].astype(np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    if skip:
        return None, len(got), False
    after = None if close else pool.state[slot].double().cpu().numpy()
    eo, ef = step_errors(st, ref, got, after, pool, fr_peak)
    worst = max([e for e in (eo, ef) if e is not None], default=0.0)
    tol = TOL_ONE if K <= 1 else TOL_ITER
    if worst > tol:
        st2 = st0.copy()
        ref2 = perturbed_step(st2, mags64, close, K, de, seed=len(got) + 7 * st0.c)
        spread = 0.0
        if len(ref):
            spread = max(spread, float(np.abs(ref2 - ref).max() / max(np.abs(ref).max(), fr_peak, 1e-300)))
        if not close and st.nbuf:
            pk = max(np.abs(v).max() for v in st.fr.values())
            spread = max(spread, max(float(np.abs(st2.fr[F] - st.fr[F]).max() / pk) for F in st.fr))
        assert spread > tol, ("error beyond the bound on a well-conditioned step", worst, spread)
        return 0.0, len(got), True
    return worst, len(got), False


def grid_cases():
    """Every (win, hop) at every look-ahead; K, de-emphasis and magnitude kind cycle so that each value meets many
    pairs, and one case runs K = 32."""
    out = []
    for i, (win, hop) in enumerate(PAIRS):
        for j, la in enumerate(LAS):
            k = i * len(LAS) + j
            K = [0, 1, 8][k % 3]
            if (win, hop, la) == (1200, 300, 3):
                K = 32
            out.append((win, hop, la, K, DEEMPHS[(k // 3) % 4], KINDS[k % 4]))
    return out


GRID = grid_cases()


@pytest.mark.parametrize("win,hop,la,K,deemph,kind", GRID,
                         ids=[f"win{w}-hop{h}-la{a}-K{k}-de{d:g}-{m}" for w, h, a, k, d, m in GRID])
def test_rtisi_steps_match_float64(win, hop, la, K, deemph, kind):
    rng = np.random.default_rng(win * 7 + hop * 3 + la)
    nb = la + 1
    T = nb + 4
    mags = make_mags(kind, win, hop, T, rng)
    pool = Pool(win, hop, la, 3)
    slot = 1
    worst = 0.0
    for f in range(T + 1):
        close = f == T
        e, _, ill = checked_step(pool, slot, mags[f:f + 1] if not close else mags[:0], close, K, deemph,
                                 skip=f == 0 and K > 1)
        assert not ill, ("a grid step was ill-conditioned", f)
        if e is not None:
            worst = max(worst, e)
    tol = TOL_ONE if K <= 1 else TOL_ITER
    print(f"\nrtisi step win={win} hop={hop} la={la} K={K} deemph={deemph:g} {kind}: worst {worst:.2e} (bound {tol:g})")
    assert worst <= tol, worst
    # the whole stream, T frames, gave hop (T - 1) samples: checked per launch by launch()
    assert tuple(int(v) for v in pool.count[slot].cpu()) == (T, 0)


# ------------------------------------------------------------------ launch splits
def run_schedule(pool, slot, mags, schedule, K, deemph, close_with_last):
    """Feed mags in launches of the sizes in schedule (0 = an empty launch), then close (in the last launch or in an
    empty one).  Returns (samples, state bits, counts)."""
    outs, f = [], 0
    for i, p in enumerate(schedule):
        last = i == len(schedule) - 1
        outs += launch(pool, K, deemph, [(slot, mags[f:f + p], last and close_with_last)])
        f += p
    assert f == len(mags)
    if not close_with_last:
        outs += launch(pool, K, deemph, [(slot, mags[:0], True)])
    return (np.concatenate(outs).view(np.uint32), pool.state[slot].cpu().numpy().view(np.uint32).copy(),
            tuple(int(v) for v in pool.count[slot].cpu()))


def split(T, p, empty_between=False):
    out, f = [], 0
    while f < T:
        out.append(min(p, T - f))
        f += out[-1]
        if empty_between:
            out.append(0)
    return out


@pytest.mark.parametrize("win,hop", PAIRS, ids=[f"win{w}-hop{h}" for w, h in PAIRS])
def test_rtisi_launch_splits_bitwise(win, hop):
    rng = np.random.default_rng(win + 13 * hop)
    for j, la in enumerate(LAS):
        nb = la + 1
        T = 2 * (2 * nb + 1) + 3
        K, deemph = [8, 1, 0, 8][j], DEEMPHS[j]
        mags = make_mags(["harmonic", "random"][j % 2], win, hop, T, rng)
        pool = Pool(win, hop, la, 4)
        ref = run_schedule(pool, 2, mags, [1] * T, K, deemph, False)
        assert len(ref[0]) == hop * (T - 1) and ref[2] == (T, 0)
        schedules = [(split(T, 1, empty_between=True), True), (split(T, nb), False), (split(T, nb), True),
                     (split(T, 2 * nb + 1), True), (split(T, 2 * nb + 1), False), ([T], True)]
        if nb > 1:
            schedules += [(split(T, nb - 1), True), (split(T, nb - 1, empty_between=True), False)]
        for sched, with_last in schedules:
            pool.state.zero_()
            pool.count.zero_()
            got = run_schedule(pool, 2, mags, sched, K, deemph, with_last)
            assert np.array_equal(got[0], ref[0]), (win, hop, la, sched, with_last, "samples")
            assert np.array_equal(got[1], ref[1]), (win, hop, la, sched, with_last, "state")
            assert got[2] == ref[2]


# ------------------------------------------------------------------ a stream's life
EDGE_PAIRS = [(1200, 300), (2048, 1024), (2046, 1023), (1200, 350), (4, 1), (2, 1)]


@pytest.mark.parametrize("win,hop", EDGE_PAIRS)
def test_rtisi_stream_edges(win, hop):
    """Closes at T = 0, T = 1, T < nb (nothing committed before the close) and right after a commit, each checked
    against the float64 restatement and for hop (T - 1) samples in all."""
    rng = np.random.default_rng(win + hop)
    worst, n_ill = 0.0, 0
    for la in (0, 1, 3, 7):
        nb = la + 1
        pool = Pool(win, hop, la, 2)
        for T, how in [(0, "empty close"), (1, "frame, then close"), (1, "frame and close together"),
                       (min(nb - 1, 3), "T < nb"), (nb, "close right after a commit"),
                       (nb + 2, "close right after a commit")]:
            if how == "T < nb" and T < 1:
                continue
            pool.state.zero_()
            pool.count.zero_()
            mags = make_mags("harmonic", win, hop, max(T, 1), rng)[:T]
            total = 0
            if how == "frame and close together":
                total += len(launch(pool, 1, 0.97, [(0, mags, True)])[0])
            else:
                for f in range(T):
                    e, n, ill = checked_step(pool, 0, mags[f:f + 1], False, 1, 0.97)
                    worst, total, n_ill = max(worst, e), total + n, n_ill + ill
                if how.startswith("close right after"):
                    assert int(pool.count[0, 0]) == T - la      # the last frame committed one
                e, n, ill = checked_step(pool, 0, mags[:0], True, 1, 0.97)
                worst, total, n_ill = max(worst, e), total + n, n_ill + ill
            assert total == hop * max(T - 1, 0), (la, T, how, total)
            assert int(pool.count[0, 0]) == T and int(pool.count[0, 1]) == 0
    print(f"\nrtisi edges win={win} hop={hop}: worst {worst:.2e} (bound {TOL_ONE:g}), {n_ill} ill-conditioned steps")
    assert worst <= TOL_ONE, worst
    assert n_ill == 0 or win == 4, "only the 4-sample window's first steps are ill-conditioned"


# ------------------------------------------------------------------ many streams
def test_rtisi_many_streams_bitwise():
    win, hop, la, K, deemph = 1200, 300, 3, 2, 0.97
    n_streams, n_slots = 1024, 1600
    rng = np.random.default_rng(5)
    pool = Pool(win, hop, la, n_slots)
    nan_state = torch.full((pool.stride,), float(STATE_NAN), device=DEV)
    pool.state.copy_(nan_state.expand(n_slots, -1))
    pool.count.copy_(torch.tensor([-7, 12345], dtype=torch.int32, device=DEV).expand(n_slots, -1))
    slots = rng.permutation(n_slots)[:n_streams]
    # random phases: each stream has had 0 to 9 frames in two launches of its own sizes
    pool.state[torch.from_numpy(slots).to(DEV)] = 0.0
    pool.count[torch.from_numpy(slots).to(DEV)] = 0
    for _ in range(2):
        ps = rng.integers(0, 6, n_streams)
        launch(pool, K, deemph, [(int(s), rng.uniform(0, 2, (p, NBIN)), False) for s, p in zip(slots, ps)])
    idle = np.setdiff1d(np.arange(n_slots), slots)
    idle_before = (pool.state[idle].cpu().numpy().view(np.uint32).copy(), pool.count[idle].cpu().numpy().copy())
    snaps = {int(s): pool.snapshot(int(s)) for s in slots}
    ps = rng.integers(0, 6, n_streams)
    closes = rng.random(n_streams) < 0.25
    mags = [rng.uniform(0, 2, (p, NBIN)).astype(np.float32) for p in ps]
    entries = [(int(s), m, bool(c)) for s, m, c in zip(slots, mags, closes)]
    outs = launch(pool, K, deemph, entries)
    after = {int(s): pool.snapshot(int(s)) for s in slots}
    assert np.array_equal(pool.state[idle].cpu().numpy().view(np.uint32), idle_before[0])
    assert np.array_equal(pool.count[idle].cpu().numpy(), idle_before[1])
    cs = pool.count[torch.from_numpy(slots).to(DEV)].cpu().numpy()
    print(f"\n{n_streams} streams: committed counts {cs[:, 0].min()}..{cs[:, 0].max()}, "
          f"{int(closes.sum())} closes, {sum(len(o) for o in outs)} samples")
    for i in rng.choice(n_streams, 24, replace=False):
        s = int(slots[i])
        pool.restore(s, snaps[s])
        alone = launch(pool, K, deemph, [entries[i]])[0]
        assert np.array_equal(alone.view(np.uint32), outs[i].view(np.uint32)), i
        assert torch.equal(pool.state[s].view(torch.int32), after[s][0].view(torch.int32)), i
        assert torch.equal(pool.count[s], after[s][1]), i


# ------------------------------------------------------------------ argument checks
def test_rtisi_state_floats():
    lib = L.load()
    for win in (2, 4, 300, 1200, 2046, 2048):
        for la in range(8):
            nb = la + 1
            assert lib.avc_rtisi_state_floats(win, la) == (nb * win + nb * NBIN + win + 1 + 3) // 4 * 4
    for win, la in [(0, 3), (-2, 3), (1200, -1), (0, -1)]:
        assert lib.avc_rtisi_state_floats(win, la) == 0


def test_rtisi_argument_checks():
    lib = L.load()
    pool = Pool(1200, 300, 3, 2)
    mag = torch.zeros(2, NBIN, device=DEV)
    i32 = torch.tensor([0, 1, 0, 0], dtype=torch.int32, device=DEV)
    out_off = torch.zeros(1, dtype=torch.int64, device=DEV)
    y = torch.zeros(16, device=DEV)
    INVALID, UNSUPPORTED = L.ERR_INVALID, L.ERR_UNSUPPORTED
    s = stream()
    n0 = L.launch_count()

    def good():
        return rtisi_desc(pool, 2, 0.97, 1, mag, i32, out_off, y)

    cases = [(dict(n_fft=1024), UNSUPPORTED, "only n_fft = 2048"),
             (dict(win=1201), UNSUPPORTED, "win must be even"), (dict(win=0), UNSUPPORTED, "win must be even"),
             (dict(win=-2), UNSUPPORTED, "win must be even"), (dict(win=2050), UNSUPPORTED, "win must be even"),
             (dict(hop=0), UNSUPPORTED, "hop must be in (0, win/2]"),
             (dict(hop=601), UNSUPPORTED, "hop must be in (0, win/2]"),
             (dict(lookahead=-1), UNSUPPORTED, "lookahead must be in [0, 7]"),
             (dict(lookahead=8), UNSUPPORTED, "lookahead must be in [0, 7]"),
             (dict(n_iter=-1), INVALID, "n_iter < 0"), (dict(n_streams=-1), INVALID, "n_streams < 0"),
             (dict(deemph=float("nan")), INVALID, "not finite"), (dict(deemph=float("inf")), INVALID, "not finite"),
             (dict(deemph=float("-inf")), INVALID, "not finite")]
    cases += [({k: None}, INVALID, "null pointer")
              for k in ("mag", "mag_off", "slot", "close", "out_off", "y", "state", "count")]
    for change, code, text in cases:
        d = good()
        for k, v in change.items():
            setattr(d, k, v)
        rc = lib.avc_rtisi_la(C.byref(d), s)
        assert rc == code and text in L.last_error(), (change, rc, L.last_error())
    rc = lib.avc_rtisi_la(None, s)
    assert rc == INVALID and "null descriptor" in L.last_error()
    assert L.launch_count() == n0
    # no streams: nothing to read, nothing launched, whatever the pointers
    d = L.RtisiDesc(n_fft=NFFT, hop=300, win=1200, lookahead=3, n_iter=2, n_streams=0, deemph=0.97)
    assert lib.avc_rtisi_la(C.byref(d), s) == 0
    assert L.launch_count() == n0
    # the checks left the library and the pool usable
    launch(pool, 2, 0.97, [(0, mag[:1].cpu().numpy(), False)])
    assert L.launch_count() == n0 + 1


# ------------------------------------------------------------------ past 2^31 samples
def shifted_pair(win, hop, la, c0, delta, runup=True, seed=0):
    """A pool whose slots 0 and 1 hold the same state, with counts (c0, nbuf) and (c0 + delta, nbuf): a run-up of
    c0 + nbuf frames or random contents."""
    nb = la + 1
    assert delta % nb == 0, "frames sit at slot F mod nb"
    rng = np.random.default_rng(seed)
    pool = Pool(win, hop, la, 4)
    nbuf = la
    if runup:
        mags = harmonic_mags(win, hop, c0 + nbuf, seed)
        launch(pool, 2, 0.97, [(0, mags, False)])
    else:
        pool.state[0] = torch.from_numpy(rng.standard_normal(pool.stride).astype(np.float32) * 0.01).to(DEV)
        pool.count[0] = torch.tensor([c0, nbuf], dtype=torch.int32)
    assert tuple(int(v) for v in pool.count[0].cpu()) == (c0, nbuf)
    for k in (1, 2, 3):
        pool.state[k] = pool.state[0]
    pool.count[1] = pool.count[3] = torch.tensor([c0 + delta, nbuf], dtype=torch.int32)
    pool.count[2] = pool.count[0]
    return pool


def straddle_delta(target, c0, hop, nb, before):
    """The delta = 0 mod nb whose shifted counts put sample c hop at `before` frames before target."""
    c1 = target // hop - before
    return (c1 - c0) // nb * nb


INVARIANCE = [  # (win, hop, la, c0, target sample (or frame at hop 1), frames before it, run-up)
    (1200, 300, 3, 8, 2 ** 31, 2, True),             # the launch's positions straddle 2^31
    (1200, 300, 3, 8, 2 ** 32 + 10 ** 6, 0, True),   # past 2^32
    (2048, 1024, 7, 4, 2 ** 31, 4, True),
    (2046, 1023, 1, 6, 2 ** 31 + 5 * 2 ** 30, 1, False),   # past 2^32, random state
    (1200, 350, 0, 8, 2 ** 31, 1, True),
    (4, 1, 3, 8, 2 ** 31 - 1, 20, True),             # hop 1: c + nbuf just below 2^31 frames
]


@pytest.mark.parametrize("win,hop,la,c0,target,before,runup", INVARIANCE,
                         ids=[f"win{c[0]}-hop{c[1]}-la{c[2]}-{c[4]}" for c in INVARIANCE])
def test_rtisi_translation_invariance(win, hop, la, c0, target, before, runup):
    nb = la + 1
    delta = straddle_delta(target, c0, hop, nb, before)
    pool = shifted_pair(win, hop, la, c0, delta, runup, seed=win + hop)
    p = 2 * nb + 1
    mags = harmonic_mags(win, hop, p, seed=99)
    c1 = c0 + delta
    assert c1 + la + p <= 2 ** 31 - 1      # frame counts are int32
    lo, hi = c1 * hop - win // 2, (c1 + la + p) * hop + win // 2
    print(f"\nshifted by {delta} frames: samples {lo} .. {hi}")
    outs = launch(pool, 8, 0.97, [(0, mags, False), (1, mags, False), (2, mags, True), (3, mags, True)])
    for a, b in ((0, 1), (2, 3)):
        assert len(outs[a]) == len(outs[b]) > 0
        assert np.array_equal(outs[a].view(np.uint32), outs[b].view(np.uint32)), (a, b)
        assert torch.equal(pool.state[a].view(torch.int32), pool.state[b].view(torch.int32)), (a, b)
        ca, cb = pool.count[a].cpu().numpy(), pool.count[b].cpu().numpy()
        assert ca[0] + delta == cb[0] and ca[1] == cb[1], (ca, cb)


def test_rtisi_shifted_step_matches_float64():
    """Steps of a state shifted across 2^31 samples against the restatement, which keeps positions as Python ints."""
    win, hop, la = 1200, 300, 3
    delta = straddle_delta(2 ** 31, 8, hop, la + 1, 2)
    pool = shifted_pair(win, hop, la, 8, delta, True, seed=3)
    mags = harmonic_mags(win, hop, 3, seed=4)
    worst = 0.0
    for f in range(3):
        e, _, ill = checked_step(pool, 1, mags[f:f + 1], False, 1, 0.97)
        assert not ill
        worst = max(worst, e)
    e, _, ill = checked_step(pool, 1, mags[:0], True, 1, 0.97)
    assert not ill
    worst = max(worst, e)
    assert int(pool.count[1, 0]) == 8 + delta + la + 3
    print(f"\nrtisi shifted step (sample {(8 + delta) * hop}): worst {worst:.2e}")
    assert worst <= TOL_ONE, worst


# ------------------------------------------------------------------ windowed STFT
def window_first(o, win, hop):
    """avc_stft_window's first sample of an entry with origin o."""
    return max(0, o * hop - win // 2 - 2)


def stft_table(entries, win, hop, gap=23):
    """An origin table of entries [(samples float32, origin, n_frames)] with NaN gaps between them: (table, y, rows)."""
    tab = np.zeros(len(entries), _SEG)
    pos, foff, parts = gap, 0, [np.full(gap, GAP_NAN, np.float32)]
    for k, (y, o, n) in enumerate(entries):
        tab[k] = (pos, len(y), foff, n, o)
        parts += [np.asarray(y, np.float32), np.full(gap, GAP_NAN, np.float32)]
        pos += len(y) + gap
        foff += n
    return torch.from_numpy(tab.view(np.uint8)).to(DEV), np.concatenate(parts), foff


def stft_call(fn, table, n_seg, y, rows, win, hop, mode, pe, outs):
    """avc_stft / avc_stft_window; outs: the output fields, each a guarded NaN-filled buffer.  Returns their bits."""
    yg = Guarded(len(y), y)
    g = {k: Guarded(rows * NBIN * (2 if k == "X" else 1), np.full(rows * NBIN * (2 if k == "X" else 1), np.nan,
                                                                   np.float32)) for k in outs}
    d = L.AudioDesc(n_fft=NFFT, hop=hop, win=win, n_seg=n_seg, n_frames=rows, n_samples=len(y), mode=mode,
                    preemph=pe, max_db=100.0, ref_db=20.0, segs=_ptr(table), y=_ptr(yg.t),
                    **{k: _ptr(v.t) for k, v in g.items()})
    L.check(getattr(L.load(), fn)(C.byref(d), stream()), fn)
    torch.cuda.synchronize()
    yg.check(fn + " y")
    assert np.array_equal(yg.np().view(np.uint32), np.asarray(y, np.float32).view(np.uint32)), "input modified"
    for k, v in g.items():
        v.check(f"{fn} {k}")
    return {k: bits(v.t).reshape(rows, -1) for k, v in g.items()}


MODES = [("MAG", ("mag_out", "mag_db")), ("MAG", ("mag_out",)), ("MAG", ("mag_db",)), ("COMPLEX", ("X",))]


@pytest.mark.parametrize("win,hop", STFT_PAIRS, ids=[f"win{w}-hop{h}" for w, h in STFT_PAIRS])
def test_stft_window_matches_stft(win, hop):
    """Entries at random origins, closed (the end reflects) and still arriving (frames inside the entry only), several
    per signal in one ragged table: each frame has avc_stft's bits for the whole signal."""
    lengths = stft_lengths(hop)[:4]
    ys = signals(lengths, 200 + win + hop)
    rng = np.random.default_rng(win + hop)
    for pe in (0.0, float(np.float32(0.97))):
        for mode, fields in MODES:
            m = getattr(L, "STFT_" + mode)
            whole = []
            for y in ys:
                tab, yy, rows = stft_table([(y, 0, 1 + len(y) // hop)], win, hop)
                whole.append(stft_call("avc_stft", tab, 1, yy, rows, win, hop, m, pe, fields))
            entries, want = [], []
            for y, ref in zip(ys, whole):
                T = 1 + len(y) // hop
                for o in sorted({o for o in {0, 1, T - 1} | set(rng.integers(0, T, 4).tolist()) if o < T}):
                    k = int(rng.integers(1, T - o + 1))
                    if o + k == T:                      # closed: the entry runs to the signal's end
                        entries.append((y[window_first(o, win, hop):], o, k))
                    else:                               # arriving: it ends after the last frame's window
                        end = (o + k - 1) * hop + win // 2
                        if end > len(y):
                            continue
                        entries.append((y[window_first(o, win, hop):end], o, k))
                    want.append({f: v[o:o + k] for f, v in ref.items()})
            tab, yy, rows = stft_table(entries, win, hop)
            got = stft_call("avc_stft_window", tab, len(entries), yy, rows, win, hop, m, pe, fields)
            r = 0
            for (_, o, k), w in zip(entries, want):
                for f in fields:
                    assert np.array_equal(got[f][r:r + k], w[f]), (win, hop, pe, mode, f, o, k)
                r += k


STFT_SHIFTS = [(1200, 300), (2046, 1023), (2048, 7)]


@pytest.mark.parametrize("win,hop", STFT_SHIFTS, ids=[f"win{w}-hop{h}" for w, h in STFT_SHIFTS])
def test_stft_window_translation_invariance(win, hop):
    """An interior entry (no reflection at sample 0) and one ending at a closed stream's end reflection give the same
    bits at origin o0 and o0 + delta, with o hop past 2^31 and past 2^32."""
    y = signals([40 * hop + 4 * NFFT], 7)[0]
    o0 = win // hop + 3
    first0 = window_first(o0, win, hop)
    assert first0 > 0
    k = 12
    interior = y[first0:(o0 + k - 1) * hop + win // 2]
    closed = y[first0:]
    k_closed = 1 + (len(y)) // hop - o0
    for pe in (0.0, float(np.float32(0.97))):
        for mode, fields in (("MAG", ("mag_out", "mag_db")), ("COMPLEX", ("X",))):
            m = getattr(L, "STFT_" + mode)
            for target in (2 ** 31, 2 ** 32 + 12345):
                o1 = target // hop - 3
                entries = [(interior, o0, k), (interior, o1, k), (closed, o0, k_closed), (closed, o1, k_closed)]
                tab, yy, rows = stft_table(entries, win, hop)
                got = stft_call("avc_stft_window", tab, len(entries), yy, rows, win, hop, m, pe, fields)
                for f in fields:
                    a = got[f]
                    assert np.array_equal(a[:k], a[k:2 * k]), (pe, mode, f, target, "interior")
                    assert np.array_equal(a[2 * k:2 * k + k_closed], a[2 * k + k_closed:]), (pe, mode, f, target)
                    assert not np.isnan(a.view(np.float32)).any()


def test_yin_window_translation_invariance():
    """avc_yin_window: the same entries at o0 and o0 + delta, o hop past 2^31 and 2^32, interior and closed."""
    from adaptive_voice_conversion_b200 import f0 as F
    from test_gpu_stream_pitch import HOP, SR, first, yin_window
    p = F.F0Params()
    span = p.win + p.tau_max(SR)
    y = torch.from_numpy(signals([60 * HOP + 4 * span], 9)[0]).to(DEV)
    o0 = span // HOP + 3
    assert first(o0) > 0
    k = 10
    interior = y[first(o0):(o0 + k - 1) * HOP + span - span // 2]
    closed = y[first(o0):]
    k_closed = 1 + y.numel() // HOP - o0
    for target in (2 ** 31, 2 ** 32 + 777):
        o1 = target // HOP - 2
        got = yin_window([(interior, o0, k), (interior, o1, k), (closed, o0, k_closed), (closed, o1, k_closed)])
        assert not np.isnan(got[0]).any() and not np.isnan(got[2]).any()
        assert np.array_equal(got[0], got[1]) and np.array_equal(got[2], got[3]), target
