"""Griffin-Lim vocoder on the GPU: the reference's wav <-> mel DSP (preprocess/tacotron/utils.py get_spectrograms,
melspectrogram2wav, with its hyperparams.py) on the kernels of csrc/audio.cu.

The semantics follow librosa 0.6/0.7 (the releases of the reference's PyTorch 1.0.1): periodic Hann window of
win_length centred in n_fft, center=True reflect-padded STFT, iSTFT normalised by the window sum-square, the Slaney
mel filterbank (htk=False, norm=1) and its pseudo-inverse as the reference builds it, and librosa.effects.trim.
oracle/audio_oracle.py restates every definition in float64.  A file that is not at ``sr`` is resampled with
scipy.signal.resample_poly; librosa used resampy, so such input does not match the reference bit for bit.

Every stage function takes a ragged batch, a list of device tensors of different lengths, and converts it with one
launch per kernel.  No kernel uses atomics, so each utterance gets the bits it gets when converted alone.
``Vocoder`` has the duck type ``Inferencer`` accepts (``get_spectrograms(path)``, ``melspectrogram2wav(mel)``, numpy
in and out) and the batched device forms ``wav_to_mel`` / ``mel_to_wav`` (``mel_to_signal`` leaves the synthesis
untrimmed, aligned with the mel frames).  ``pitch_shift`` transposes the linear magnitudes before Griffin-Lim
(``AudioParams.pitch_shift`` or ``semitones=``, per utterance or per frame), keeping the frame grid.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, replace
from math import gcd

import numpy as np
import torch

from . import _lib as L
from .utils import _stream, local_device

TRIM_FRAME, TRIM_HOP = 2048, 512   # librosa.effects.trim defaults


@dataclass(frozen=True)
class AudioParams:
    """The reference's tacotron hyper-parameters (n_mels is the model's c_in)."""
    sr: int = 24000
    n_fft: int = 2048
    hop_length: int = 300
    win_length: int = 1200
    n_mels: int = 512
    n_iter: int = 100
    momentum: float = 0.0      # fast Griffin-Lim momentum in [0, 1); 0 is the reference's plain Griffin-Lim
    gl_init: str = "zero"      # Griffin-Lim start phase: "zero" (the reference's) or "pghi" (phase-gradient estimate)
    pghi_tol: float = 1e-5     # PGHI significance threshold relative to an utterance's largest magnitude (not tuned)
    pitch_shift: float = 0.0   # semitones in [-24, 24] applied to the synthesis (formant-preserving, ``pitch_shift``)
    ps_lifter: int = 40        # cepstral lifter of the shift's envelope: not tuned, below the 48-sample period of 500 Hz
    preemphasis: float = 0.97
    max_db: float = 100.0
    ref_db: float = 20.0
    top_db: float = 15.0       # trim of the input wav
    out_top_db: float = 60.0   # trim of the synthesised wav (librosa's default)

    @property
    def n_bins(self) -> int:
        return self.n_fft // 2 + 1

    @property
    def min_samples(self) -> int:
        """Shortest signal an STFT accepts: its reflect padding of n_fft/2 must not wrap around twice."""
        return self.n_fft // 2 + 1

    @property
    def min_frames(self) -> int:
        """Fewest mel frames whose iSTFT is long enough to be re-analysed."""
        return 1 + -(-self.min_samples // self.hop_length)


# ------------------------------------------------------------------ host-side tables (float64)
def hz_to_mel(f):
    """Slaney scale: f / (200/3) below 1 kHz, 15 + ln(f / 1000) / (ln 6.4 / 27) above."""
    f = np.asarray(f, np.float64)
    return np.where(f >= 1000.0, 15.0 + np.log(np.maximum(f, 1000.0) / 1000.0) / (np.log(6.4) / 27.0), f * 3.0 / 200.0)


def mel_to_hz(m):
    m = np.asarray(m, np.float64)
    return np.where(m >= 15.0, 1000.0 * np.exp((np.log(6.4) / 27.0) * (np.maximum(m, 15.0) - 15.0)), m * 200.0 / 3.0)


def mel_filterbank(hp: AudioParams) -> np.ndarray:
    """librosa.filters.mel(sr, n_fft, n_mels), fmin 0, fmax sr/2: [n_mels, n_bins] float64.  With many mels the
    lowest filters fall between FFT bins and are empty."""
    fft_f = np.linspace(0.0, hp.sr / 2.0, hp.n_bins)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(0.0), hz_to_mel(hp.sr / 2.0), hp.n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fft_f[None, :]
    lower = -ramps[:-2] / fdiff[:-1, None]
    upper = ramps[2:] / fdiff[1:, None]
    return np.maximum(0.0, np.minimum(lower, upper)) * (2.0 / (mel_f[2:] - mel_f[:-2]))[:, None]


def mel_to_linear_matrix(fb: np.ndarray) -> np.ndarray:
    """The reference's pseudo-inverse M = fb^T diag(d), d_j = 1/colsum_j(fb fb^T) (the colsum where |colsum| <= 1e-8,
    i.e. for the empty filters): [n_bins, n_mels]."""
    cs = (fb @ fb.T).sum(axis=0)
    d = np.where(np.abs(cs) > 1e-8, 1.0 / np.where(cs == 0, 1.0, cs), cs)
    return fb.T * d[None, :]


def read_pcm(path: str):
    """(rate, samples) of a wav file as stored: [n] or [n, channels], the file's own sample type."""
    from scipy.io import wavfile
    return wavfile.read(path)


def scale_pcm(data: np.ndarray) -> np.ndarray:
    """PCM samples as float64: integer PCM scaled to [-1, 1), float PCM as is."""
    if data.dtype.kind == "i":
        y = data / float(2 ** (8 * data.dtype.itemsize - 1))
    elif data.dtype.kind == "u":
        half = float(2 ** (8 * data.dtype.itemsize - 1))
        y = (data - half) / half
    else:
        y = data.astype(np.float64)
    return y


def load_wav(path: str, sr: int) -> np.ndarray:
    """A wav file as float32 mono at sr: channels averaged, integer PCM scaled to [-1, 1), resampled with
    scipy.signal.resample_poly when the file has another rate."""
    from scipy.signal import resample_poly
    rate, data = read_pcm(path)
    y = scale_pcm(data)
    if y.ndim == 2:
        y = y.mean(axis=1)
    if rate != sr:
        g = gcd(int(rate), int(sr))
        y = resample_poly(y, sr // g, rate // g)
    return np.ascontiguousarray(y, np.float32)


# ------------------------------------------------------------------ ragged batches
_SEG = np.dtype([("sample_off", "<i8"), ("n_samples", "<i4"), ("frame_off", "<i4"), ("n_frames", "<i4"),
                 ("reserved", "<i4")])
assert _SEG.itemsize == C.sizeof(L.AudioSeg)


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


class _Ragged:
    """Utterances laid end to end: the device table of per-utterance sample and frame offsets, and with origins each
    entry's frame origin (``reserved``: the absolute index of its first frame, for the windowed kernels)."""

    def __init__(self, n_samples, n_frames, dev, origins=None):
        self.n_samples, self.n_frames = [int(n) for n in n_samples], [int(n) for n in n_frames]
        self.sample_offs = np.concatenate([[0], np.cumsum(self.n_samples)]).astype(np.int64)
        self.frame_offs = np.concatenate([[0], np.cumsum(self.n_frames)]).astype(np.int64)
        if self.frame_offs[-1] >= 2 ** 31 or self.sample_offs[-1] >= 2 ** 31:
            raise ValueError("ragged batch too large: split it (2^31 frames or samples at most)")
        tab = np.zeros(len(self.n_samples), _SEG)
        tab["sample_off"], tab["n_samples"] = self.sample_offs[:-1], self.n_samples
        tab["frame_off"], tab["n_frames"] = self.frame_offs[:-1], self.n_frames
        if origins is not None:
            tab["reserved"] = origins
        self.table = torch.from_numpy(tab.view(np.uint8)).to(dev)

    def desc(self, hp: AudioParams, **kw) -> L.AudioDesc:
        d = L.AudioDesc(n_fft=hp.n_fft, hop=hp.hop_length, win=hp.win_length, n_seg=len(self.n_samples),
                        n_frames=int(self.frame_offs[-1]), n_samples=int(self.sample_offs[-1]),
                        max_db=hp.max_db, ref_db=hp.ref_db, segs=_ptr(self.table))
        for k, v in kw.items():
            setattr(d, k, _ptr(v) if isinstance(v, torch.Tensor) or v is None else v)
        return d

    def split_samples(self, y):
        return list(torch.split(y, self.n_samples))

    def split_frames(self, x):
        return list(torch.split(x, self.n_frames))


def _signals(wavs, hp: AudioParams, what: str):
    ys = [w.reshape(-1).float().contiguous() for w in wavs]
    if not ys:
        raise ValueError(f"{what}: empty batch")
    for i, y in enumerate(ys):
        if y.numel() < hp.min_samples:
            raise ValueError(f"{what}: utterance {i} has {y.numel()} samples; an STFT with n_fft={hp.n_fft} needs at "
                             f"least {hp.min_samples}")
    return ys


def _call(fn, desc, dev, *extra):
    L.check(getattr(L.load(), fn)(C.byref(desc), *extra, _stream(dev)), fn)


# ------------------------------------------------------------------ stages
def stft(wavs, hp: AudioParams = AudioParams(), preemphasis: float = 0.0):
    """Half spectra [1 + n//hop, n_bins] complex64 of each signal (pre-emphasis applied on the fly when non-zero)."""
    ys = _signals(wavs, hp, "stft")
    dev = ys[0].device
    r = _Ragged([y.numel() for y in ys], [1 + y.numel() // hp.hop_length for y in ys], dev)
    X = torch.empty(int(r.frame_offs[-1]), hp.n_bins, 2, device=dev)
    _call("avc_stft", r.desc(hp, mode=L.STFT_COMPLEX, preemph=preemphasis, y=torch.cat(ys), X=X), dev)
    return [torch.view_as_complex(x) for x in r.split_frames(X)]


def magnitude(wavs, hp: AudioParams = AudioParams(), preemphasis: float = 0.0):
    """(|STFT|, its normalised dB) per signal: the analysis epilogue of the STFT kernel."""
    ys = _signals(wavs, hp, "magnitude")
    dev = ys[0].device
    r = _Ragged([y.numel() for y in ys], [1 + y.numel() // hp.hop_length for y in ys], dev)
    mag = torch.empty(int(r.frame_offs[-1]), hp.n_bins, device=dev)
    mag_db = torch.empty_like(mag)
    _call("avc_stft", r.desc(hp, mode=L.STFT_MAG, preemph=preemphasis, y=torch.cat(ys), mag_out=mag, mag_db=mag_db), dev)
    return list(zip(r.split_frames(mag), r.split_frames(mag_db)))


def _frames(specs, hp: AudioParams, what: str):
    for i, s in enumerate(specs):
        if s.shape[0] < hp.min_frames:
            raise ValueError(f"{what}: utterance {i} has {s.shape[0]} frames; at least {hp.min_frames} are needed "
                             f"(hop * (frames - 1) >= n_fft/2 + 1 samples)")
    if not specs:
        raise ValueError(f"{what}: empty batch")


def istft(specs, hp: AudioParams = AudioParams()):
    """Signals of hop * (T - 1) samples from half spectra [T, n_bins] (complex, or real = zero phase)."""
    _frames(specs, hp, "istft")
    dev = specs[0].device
    r = _Ragged([hp.hop_length * (s.shape[0] - 1) for s in specs], [s.shape[0] for s in specs], dev)
    cplx = torch.is_complex(specs[0])
    spec = torch.cat([torch.view_as_real(s) if cplx else s for s in specs]).float().contiguous()
    frames = torch.empty(int(r.frame_offs[-1]), hp.win_length, device=dev)
    y = torch.empty(int(r.sample_offs[-1]), device=dev)
    _call("avc_istft", r.desc(hp, X=spec if cplx else None, mag=None if cplx else spec, frames=frames, y=y), dev)
    return r.split_samples(y)


GL_INITS = ("zero", "pghi")


def _init(init, hp: AudioParams) -> str:
    init = hp.gl_init if init is None else init
    if init not in GL_INITS:
        raise ValueError(f"griffin_lim: init must be one of {GL_INITS} (got {init!r})")
    return init


def pghi(mags, hp: AudioParams = AudioParams(), tol: float | None = None, parent: bool = False):
    """Phase Gradient Heap Integration start spectra: [T, n_bins] complex64 S e^{i phi} per utterance of linear
    magnitudes S [T, n_bins], in one avc_pghi launch.  phi is integrated frame by frame from the phase derivatives the
    Gaussian approximation of the window gives from ln S (Prusa, Balazs & Sondergaard 2017; Prusa & Holighaus 2017);
    bins below ``tol`` (default ``hp.pghi_tol``) times the utterance's largest magnitude get phase 0.
    ``parent=True`` also returns each bin's int8 AVC_PGHI_* source, per utterance."""
    if not mags:
        raise ValueError("pghi: empty batch")
    dev = mags[0].device
    S = torch.cat([m.float() for m in mags]).contiguous()
    if S.dim() != 2 or S.shape[1] != hp.n_bins:
        raise ValueError(f"pghi: magnitudes have shape {tuple(S.shape)}, n_fft={hp.n_fft} gives {hp.n_bins} bins")
    r = _Ragged([0] * len(mags), [m.shape[0] for m in mags], dev)
    X = torch.empty(S.shape[0], hp.n_bins, 2, device=dev)
    par = torch.empty(S.shape[0], hp.n_bins, dtype=torch.int8, device=dev) if parent else None
    tol = float(hp.pghi_tol if tol is None else tol)
    _call("avc_pghi", r.desc(hp, mag=S, X=X), dev, C.c_float(tol), _ptr(par))
    out = [torch.view_as_complex(x) for x in r.split_frames(X)]
    return (out, r.split_frames(par)) if parent else out


class GriffinLim:
    """One ragged Griffin-Lim call with its buffers.  ``run()`` enqueues the whole loop (3 n_iter + 2 launches, one
    more with the PGHI start) on the current stream, so it can be captured into a CUDA graph; ``outputs()`` are views
    of the signal buffer.

    ``momentum`` m > 0 (default ``hp.momentum``) runs fast Griffin-Lim (Perraudin, Balazs & Sondergaard 2013) in the
    form of librosa's and torchaudio's ``momentum``: each projection uses A = E - m/(1+m) P, P the previous iteration's
    spectrum E, and P takes a second complex buffer the size of X.  The start is zero-phase (librosa's init=None).
    Where librosa divides by |A| + tiny, this divides by max(1e-8, |A|); the two differ only where |A| < 1e-8.
    A momentum that is not finite or outside [0, 1) raises ``AvcError`` from ``run()``.

    ``init`` (default ``hp.gl_init``) picks the start phase: "zero" (the reference's, and librosa's init=None), or
    "pghi", which first writes ``pghi``'s start spectrum into X (tolerance ``hp.pghi_tol``) and starts the loop's
    first iSTFT from it.  It composes with ``momentum``.  Either way ``run()`` is one C call
    (``avc_griffin_lim_from``) that checks every argument, the tolerance included, before its first launch."""

    def __init__(self, mags, hp: AudioParams = AudioParams(), n_iter: int | None = None,
                 momentum: float | None = None, init: str | None = None):
        self.init = _init(init, hp)
        self.tol = float(hp.pghi_tol)
        _frames(mags, hp, "griffin_lim")
        self.dev = mags[0].device
        self.S = torch.cat([m.float() for m in mags]).contiguous()
        if self.S.shape[1] != hp.n_bins:
            raise ValueError(f"griffin_lim: magnitudes have {self.S.shape[1]} bins, n_fft={hp.n_fft} gives {hp.n_bins}")
        self.r = _Ragged([hp.hop_length * (m.shape[0] - 1) for m in mags], [m.shape[0] for m in mags], self.dev)
        n_frames = int(self.r.frame_offs[-1])
        self.X = torch.empty(n_frames, hp.n_bins, 2, device=self.dev)
        self.frames = torch.empty(n_frames, hp.win_length, device=self.dev)
        self.y = torch.empty(int(self.r.sample_offs[-1]), device=self.dev)
        m = float(hp.momentum if momentum is None else momentum)
        self.X_prev = torch.empty_like(self.X) if m > 0 else None
        self.desc = self.r.desc(hp, n_iter=hp.n_iter if n_iter is None else n_iter, momentum=m, mag=self.S, X=self.X,
                                frames=self.frames, y=self.y, X_prev=self.X_prev)

    def run(self):
        if self.init == "pghi":
            _call("avc_griffin_lim_from", self.desc, self.dev, C.c_int32(L.GL_START_PGHI), C.c_float(self.tol))
        else:
            _call("avc_griffin_lim", self.desc, self.dev)
        return self

    def outputs(self):
        return self.r.split_samples(self.y)


def griffin_lim(mags, hp: AudioParams = AudioParams(), n_iter: int | None = None, momentum: float | None = None,
                init: str | None = None):
    """Griffin-Lim from linear magnitudes [T, n_bins]; signals of hop * (T - 1) samples (untrimmed).  ``momentum``
    and ``init`` (defaults ``hp.momentum``, ``hp.gl_init``) as in ``GriffinLim``."""
    return GriffinLim(mags, hp, n_iter, momentum, init).run().outputs()


def deemphasis(wavs, coef: float = 0.97):
    """y[n] = x[n] + coef y[n-1] per signal (scipy.signal.lfilter([1], [1, -coef]))."""
    ys = [w.reshape(-1).float() for w in wavs]
    dev = ys[0].device
    r = _Ragged([y.numel() for y in ys], [0] * len(ys), dev)
    y = torch.cat(ys)
    _call("avc_deemphasis", r.desc(AudioParams(), y=y), dev, C.c_float(coef))
    return r.split_samples(y)


def frame_power(wavs):
    """Mean power of librosa.effects.trim's frames (2048 samples, hop 512, reflect-padded) per signal."""
    ys = [w.reshape(-1).float().contiguous() for w in wavs]
    for i, y in enumerate(ys):
        if y.numel() < TRIM_FRAME // 2 + 1:
            raise ValueError(f"trim: utterance {i} has {y.numel()} samples; at least {TRIM_FRAME // 2 + 1} are needed")
    dev = ys[0].device
    r = _Ragged([y.numel() for y in ys], [1 + y.numel() // TRIM_HOP for y in ys], dev)
    p = torch.empty(int(r.frame_offs[-1]), device=dev)
    hp = AudioParams(n_fft=TRIM_FRAME, hop_length=TRIM_HOP, win_length=TRIM_FRAME)
    _call("avc_frame_power", r.desc(hp, y=torch.cat(ys)), dev, _ptr(p))
    return r.split_frames(p)


def trim_bounds(power: np.ndarray, n_samples: int, top_db: float):
    """[start, end) that librosa.effects.trim(ref=np.max) keeps, from the frame powers; (0, 0) when all is silent."""
    power = np.asarray(power, np.float64)
    db = 10.0 * np.log10(np.maximum(1e-10, power)) - 10.0 * np.log10(max(1e-10, float(power.max())))
    nz = np.flatnonzero(db > -top_db)
    if nz.size == 0:
        return 0, 0
    return int(nz[0]) * TRIM_HOP, min(n_samples, (int(nz[-1]) + 1) * TRIM_HOP)


def trim(wavs, top_db: float):
    """librosa.effects.trim of each signal: frame powers on the device, one copy to the host for the edge search.
    Returns views of the inputs."""
    ys = [w.reshape(-1) for w in wavs]
    powers = frame_power(ys)
    host = torch.cat(powers).cpu().numpy()
    out, f0 = [], 0
    for y, p in zip(ys, powers):
        s, e = trim_bounds(host[f0:f0 + p.numel()], y.numel(), top_db)
        f0 += p.numel()
        out.append(y[s:e])
    return out


_trim = trim   # the name Vocoder.wav_to_mel's trim= keyword shadows


def _mel_project(x, mat, direction, hp: AudioParams):
    n_out = hp.n_bins if direction == L.MEL_TO_MAG else hp.n_mels
    x = x.float().contiguous()
    out = torch.empty(x.shape[0], n_out, device=x.device)
    d = L.MelDesc(rows=x.shape[0], n_mels=hp.n_mels, n_bins=hp.n_bins, dir=direction, max_db=hp.max_db,
                  ref_db=hp.ref_db, in_=_ptr(x), mat=_ptr(mat), out=_ptr(out))
    L.check(L.load().avc_mel_project(C.byref(d), _stream(x.device)), "avc_mel_project")
    return out


PITCH_SHIFT_MAX = 24.0   # semitones: two octaves either way


def _semitones(semitones, n: int, what: str, frames=None) -> list:
    """Shifts of n utterances from a float or one entry per utterance, an entry being a float or a 1-D array / tensor
    of one value per frame (frames[i] of them): a float per constant utterance, a float64 array per per-frame one.
    ValueError naming the utterance for a value outside [-24, 24] or not finite, or a per-frame entry of the wrong
    length."""
    if isinstance(semitones, torch.Tensor):
        semitones = semitones.detach().cpu().numpy()
    if isinstance(semitones, (list, tuple)) or (isinstance(semitones, np.ndarray) and semitones.ndim > 0):
        entries = list(semitones)     # not np.ndim: a list mixing floats and arrays is ragged
    else:
        entries = [semitones] * n
    if len(entries) != n:
        raise ValueError(f"{what}: {len(entries)} shifts for {n} utterances")
    out = []
    for i, e in enumerate(entries):
        if isinstance(e, torch.Tensor):
            e = e.detach().cpu().numpy()
        if np.ndim(e) == 0:
            v = float(e)
            bad = not np.isfinite(v) or abs(v) > PITCH_SHIFT_MAX
            out.append(v)
        else:
            v = np.asarray(e, np.float64)
            if v.ndim != 1 or frames is None or len(v) != int(frames[i]):
                want = "one per utterance" if frames is None else f"{int(frames[i])}"
                raise ValueError(f"{what}: utterance {i}: {v.shape} per-frame shifts, expected {want} frames")
            ok = np.isfinite(v) & (np.abs(v) <= PITCH_SHIFT_MAX)
            bad = not ok.all()
            if bad:
                v = f"{v[~ok][0]} at frame {int(np.flatnonzero(~ok)[0])}"
            out.append(v)
        if bad:
            raise ValueError(f"{what}: utterance {i}: pitch shift must be finite and in [-{PITCH_SHIFT_MAX:g}, "
                             f"{PITCH_SHIFT_MAX:g}] semitones (got {v})")
    return out


def _ratio(v) -> float:
    """2^(v/12) in float64: the one place a shift becomes a ratio."""
    return 2.0 ** (v / 12.0)


def pitch_shift(mags, semitones, hp: AudioParams = AudioParams()):
    """Formant-preserving pitch shift of linear magnitudes [T, n_bins] per utterance by ``semitones`` (a float, or one
    entry per utterance: a float or T values, one per frame), in one avc_pitch_shift launch: the harmonics (the
    cepstrum above ``hp.ps_lifter``) move by the ratio float32(2^(s/12)) of each frame's shift, the envelope stays,
    the frame grid and duration are unchanged.  A frame with shift 0 is copied bit for bit, and a per-frame entry of
    equal values gives the bits of that value as a float."""
    if not mags:
        raise ValueError("pitch_shift: empty batch")
    return _shift_rows(mags, _semitones(semitones, len(mags), "pitch_shift", [int(m.shape[0]) for m in mags]), hp)


def _shift_rows(mags, semitones, hp: AudioParams):
    """The avc_pitch_shift launch of pitch_shift, on shifts it does not check: semitones[i] is a float or a float64
    array of one value per frame of mags[i]."""
    lens = [int(m.shape[0]) for m in mags]
    dev = mags[0].device
    S = torch.cat([m.float() for m in mags]).contiguous()
    if S.dim() != 2 or S.shape[1] != hp.n_bins:
        raise ValueError(f"pitch_shift: magnitudes have shape {tuple(S.shape)}, n_fft={hp.n_fft} gives {hp.n_bins} bins")
    ratio = np.concatenate([np.full(T, _ratio(v), np.float64) if isinstance(v, float) else
                            np.array([_ratio(x) for x in v.tolist()], np.float64) for v, T in zip(semitones, lens)])
    ratio = torch.from_numpy(ratio.astype(np.float32)).to(dev)
    out = torch.empty_like(S)
    L.check(L.load().avc_pitch_shift(_ptr(S), _ptr(ratio), _ptr(out), S.shape[0], hp.n_bins, int(hp.ps_lifter),
                                     _stream(dev)), "avc_pitch_shift")
    return list(torch.split(out, lens))


# ------------------------------------------------------------------ the vocoder
class Vocoder:
    """The reference's get_spectrograms / melspectrogram2wav on the GPU.  The filterbank and its pseudo-inverse are
    built once in float64 and kept on the device as float32."""

    def __init__(self, n_mels: int | None = None, hp: AudioParams | None = None, device=None):
        hp = hp or AudioParams()
        self.hp = replace(hp, n_mels=int(n_mels)) if n_mels is not None else hp
        self.device = torch.device(device) if device is not None else local_device()
        fb = mel_filterbank(self.hp)
        self.fb_t = torch.from_numpy(np.ascontiguousarray(fb.T, np.float32)).to(self.device)    # [n_bins, n_mels]
        self.m_t = torch.from_numpy(np.ascontiguousarray(mel_to_linear_matrix(fb).T, np.float32)).to(self.device)

    def wav_to_mel(self, wavs, *, trim: bool = True):
        """Signals at hp.sr (device tensors) -> [(mel [T, n_mels], mag [T, n_bins])], both normalised: trim (top_db),
        pre-emphasis, |STFT|, mel projection, dB, normalisation.  trim=False analyses the signals as they are (the
        streaming analysis of streaming.py gives these frames)."""
        hp = self.hp
        ys = (_signals(_trim(wavs, hp.top_db), hp, "wav_to_mel (after trimming)") if trim else
              _signals(wavs, hp, "wav_to_mel"))
        r = _Ragged([y.numel() for y in ys], [1 + y.numel() // hp.hop_length for y in ys], self.device)
        mag = torch.empty(int(r.frame_offs[-1]), hp.n_bins, device=self.device)
        mag_db = torch.empty_like(mag)
        _call("avc_stft", r.desc(hp, mode=L.STFT_MAG, preemph=hp.preemphasis, y=torch.cat(ys), mag_out=mag,
                                 mag_db=mag_db), self.device)
        mel = _mel_project(mag, self.fb_t, L.MAG_TO_MEL, hp)
        return list(zip(r.split_frames(mel), r.split_frames(mag_db)))

    def mel_to_mag(self, mels):
        """Normalised mels [T, n_mels] -> linear magnitudes [T, n_bins]."""
        r = [m.shape[0] for m in mels]
        return list(torch.split(_mel_project(torch.cat(mels), self.m_t, L.MEL_TO_MAG, self.hp), r))

    def mel_to_signal(self, mels, n_iter: int | None = None, momentum: float | None = None, init: str | None = None,
                      what: str = "mel_to_signal", *, semitones=None):
        """Normalised mels [T, n_mels] (device tensors) -> untrimmed float32 signals of hop * (T - 1) samples, sample
        f * hop at mel frame f: amplitude, mel-to-linear, pitch shift, Griffin-Lim, de-emphasis.  ``n_iter``,
        ``momentum``, ``init`` and ``semitones`` (a float, or one entry per utterance: a float or T values, one per
        mel frame, as ``pitch_shift``) default to ``hp.n_iter``, ``hp.momentum``, ``hp.gl_init`` and
        ``hp.pitch_shift``.  With every shift 0 no shift is launched."""
        hp = self.hp
        for i, m in enumerate(mels):
            if m.dim() != 2 or m.shape[1] != hp.n_mels:
                raise ValueError(f"{what}: utterance {i} has shape {tuple(m.shape)}, expected [T, {hp.n_mels}]")
        _init(init, hp)
        _frames(mels, hp, what)
        s = _semitones(hp.pitch_shift if semitones is None else semitones, len(mels), what,
                       [int(m.shape[0]) for m in mels])
        mags = self.mel_to_mag(mels)
        if any(np.any(v != 0.0) for v in s):
            mags = pitch_shift(mags, s, hp)
        return deemphasis(griffin_lim(mags, hp, n_iter, momentum, init), hp.preemphasis)

    def mel_to_wav(self, mels, n_iter: int | None = None, momentum: float | None = None, init: str | None = None, *,
                   semitones=None):
        """``mel_to_signal`` then trim (out_top_db): the waveform a conversion writes."""
        return trim(self.mel_to_signal(mels, n_iter, momentum, init, what="mel_to_wav", semitones=semitones),
                    self.hp.out_top_db)

    def get_spectrograms(self, path):
        """The reference's get_spectrograms(fpath): (mel [T, n_mels], mag [T, n_bins]) float32 numpy."""
        y = torch.from_numpy(load_wav(path, self.hp.sr)).to(self.device)
        mel, mag = self.wav_to_mel([y])[0]
        return mel.cpu().numpy(), mag.cpu().numpy()

    def melspectrogram2wav(self, mel):
        """The reference's melspectrogram2wav(mel): mel [T, n_mels] numpy -> float32 numpy waveform."""
        m = torch.from_numpy(np.ascontiguousarray(mel, np.float32)).to(self.device)
        return self.mel_to_wav([m])[0].cpu().numpy()
