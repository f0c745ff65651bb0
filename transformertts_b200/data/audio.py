"""Audio front-end mirror of the reference's ``data/audio.py``: STFT -> 80-bin mel -> log normalisation (reference:
data/audio.py:72-92, 196-231) by the fused CUDA kernels ``ttsb_stft_mel_log`` / ``ttsb_stft_mel_log_batch``, f0 by DIO +
StoneMask (data/audio.py:146-151) by ``ttsb_pitch_dio_stonemask``, wav loading and preprocessing (data/audio.py:126-141,
154-162) on the host, resampling to ``sampling_rate`` (librosa.load's ``kaiser_best`` resampy filter, data/audio.py:126-130) by
``ttsb_resample_batch``, the ``trim_silence`` trim of leading and trailing silence (librosa.effects.trim, data/audio.py:164-169)
by ``ttsb_trim_silence_bounds``, and mel -> waveform by Griffin-Lim.  For the WORLD mel-cepstral distortion of
``evaluate_tts.py --mcep`` (no reference counterpart): WORLD's CheapTrick envelope by ``ttsb_cheaptrick`` and pysptk's sp2mc by
``ttsb_sp2mc`` (``world_mcep_batch``), and ``load_wavs``, which rebuilds recordings as ``create_training_data.py`` prepares them.
``.flac`` recordings (librosa.load reads them through libsndfile) are decoded on the GPU by ``ttsb_flac_decode_batch``
(``read_flac_batch``), a batch of files per call; the STREAMINFO's MD5 is not checked, as libsndfile does not check it.

``trim_long_silences`` (webrtcvad voice-activity detection) is not implemented: ``preprocess`` refuses it, and refuses
``trim_silence`` without ``trim_silence_top_db``.  ``load_wav`` refuses a file whose rate differs from ``sampling_rate``; such
files are read with ``read_wav`` and resampled a batch at a time with ``resample_ragged`` / ``resample_ragged_device``, as
``create_training_data.py`` does.
"""
from __future__ import annotations

import numpy as np
import torch

from .. import lib


def _hz_to_mel_slaney(f):
    f = np.asarray(f, dtype=np.float64)
    lin = f / (200.0 / 3)
    log_region = 15.0 + np.log(np.maximum(f, 1e-10) / 1000.0) / (np.log(6.4) / 27.0)
    return np.where(f >= 1000.0, log_region, lin)


def _mel_to_hz_slaney(m):
    m = np.asarray(m, dtype=np.float64)
    lin = m * (200.0 / 3)
    log_region = 1000.0 * np.exp((np.log(6.4) / 27.0) * (m - 15.0))
    return np.where(m >= 15.0, log_region, lin)


def slaney_mel_basis(sr: int, n_fft: int, n_mels: int, fmin: float, fmax: float) -> np.ndarray:
    """Area-normalised triangular Slaney filterbank (what librosa.filters.mel(htk=False, norm=1) returns, which the
    reference reaches through librosa.feature.melspectrogram at data/audio.py:73-79) -> float32 (n_mels, 1+n_fft/2).
    fmax None means sr / 2, as librosa's fmax=None."""
    if fmax is None:
        fmax = sr / 2.0
    n_bins = 1 + n_fft // 2
    bin_hz = np.arange(n_bins, dtype=np.float64) * (sr / 2.0) / (n_bins - 1)
    edges = _mel_to_hz_slaney(np.linspace(_hz_to_mel_slaney(fmin), _hz_to_mel_slaney(fmax), n_mels + 2))
    basis = np.zeros((n_mels, n_bins), dtype=np.float64)
    for m in range(n_mels):
        left, centre, right = edges[m], edges[m + 1], edges[m + 2]
        rising = (bin_hz - left) / (centre - left)
        falling = (right - bin_hz) / (right - centre)
        basis[m] = np.clip(np.minimum(rising, falling), 0.0, None) * (2.0 / (right - left))
    return basis.astype(np.float32)


def mel_band(basis: np.ndarray) -> np.ndarray:
    """Band table of a mel basis (n_mels, n_bins) -> int32 (n_mels, 2): first / past-last bin of each row's non-zero weights,
    (0, 0) for a row of zeros."""
    nz = np.asarray(basis) != 0
    first = np.argmax(nz, axis=1)
    past_last = nz.shape[1] - np.argmax(nz[:, ::-1], axis=1)
    return np.where(nz.any(axis=1)[:, None], np.stack([first, past_last], axis=1), 0).astype(np.int32)


def kaiser_best_half_window() -> np.ndarray:
    """resampy's `kaiser_best` interpolation filter (the one librosa.load(sr=...) uses at its default res_type), restated from its
    published parameters: the right half of rolloff * sinc(rolloff * z) * kaiser(2n + 1, beta), z = linspace(0, 64, n + 1),
    n = 64 zero crossings * 512 entries per crossing -> float64 (32769,).  resampy ships this table precomputed."""
    from scipy.signal.windows import kaiser
    num_zeros, num_table, beta, rolloff = 64, 512, 14.769656459379492, 0.9475937167399596
    n = num_zeros * num_table
    sinc_win = rolloff * np.sinc(rolloff * np.linspace(0, num_zeros, num=n + 1, endpoint=True))
    return kaiser(2 * n + 1, beta)[n:] * sinc_win


class TooShortToResample(ValueError):
    """A clip with no output sample to compute at the target rate."""


FLAC_SKIPPED_BLOCKS = {1: 'PADDING', 2: 'APPLICATION', 3: 'SEEKTABLE', 4: 'VORBIS_COMMENT', 5: 'CUESHEET', 6: 'PICTURE'}


class FlacStream:
    """A .flac file read but not decoded: its bytes, where its frames start, and its STREAMINFO (RFC 9639 section 8.2)."""

    def __init__(self, path, data: bytes):
        self.path, self.data = str(path), data
        name = self.path

        def need(n, what):
            if len(data) < n:
                raise ValueError(f'{name}: truncated metadata ({what} needs {n} bytes, the file has {len(data)})')
        need(4, 'the fLaC magic')
        if data[:4] != b'fLaC':
            raise ValueError(f'{name}: not a FLAC file (no fLaC magic)')
        pos, first, last = 4, True, False
        while not last:
            need(pos + 4, 'a metadata block header')
            kind, last, length = data[pos] & 0x7F, bool(data[pos] >> 7), int.from_bytes(data[pos + 1:pos + 4], 'big')
            need(pos + 4 + length, f'metadata block type {kind}')
            body = data[pos + 4:pos + 4 + length]
            if first:
                if kind != 0 or length != 34:
                    raise ValueError(f'{name}: the first metadata block is type {kind} of {length} bytes, not a 34-byte STREAMINFO')
                v = int.from_bytes(body[10:18], 'big')
                self.min_block, self.max_block = int.from_bytes(body[0:2], 'big'), int.from_bytes(body[2:4], 'big')
                self.sample_rate, self.channels = v >> 44, (v >> 41 & 7) + 1
                self.bits_per_sample, self.total_samples = (v >> 36 & 31) + 1, v & ((1 << 36) - 1)
            elif kind == 127:
                raise ValueError(f'{name}: invalid metadata block type 127')
            elif kind == 0:
                raise ValueError(f'{name}: a second STREAMINFO block')
            # PADDING, APPLICATION, SEEKTABLE, VORBIS_COMMENT, CUESHEET, PICTURE and reserved types carry nothing the decoder needs
            first = False
            pos += 4 + length
        self.frame_offset = pos
        if self.total_samples == 0:
            raise ValueError(f'{name}: STREAMINFO gives an unknown (0) total sample count, which this decoder does not support')
        if 25 <= self.bits_per_sample <= 32:
            raise ValueError(f'{name}: {self.bits_per_sample}-bit FLAC is not supported (4 to 24 bits per sample)')
        if self.bits_per_sample < 4:
            raise ValueError(f'{name}: {self.bits_per_sample} bits per sample is not supported (4 to 24 bits per sample)')
        if not 16 <= self.min_block <= self.max_block:
            raise ValueError(f'{name}: STREAMINFO block sizes {self.min_block} to {self.max_block} (need 16 <= min <= max)')
        if self.sample_rate == 0:
            raise ValueError(f'{name}: STREAMINFO sample rate 0')

    @classmethod
    def read(cls, path):
        with open(path, 'rb') as f:
            return cls(path, f.read())

    def stream_info(self):
        """The row of ttsb_flac_decode_batch's stream_info table."""
        return (self.channels, self.bits_per_sample, self.sample_rate, self.min_block, self.max_block, self.total_samples)


class FlacDecodeError(ValueError):
    """One or more streams of a FLAC batch are malformed; `failed` maps each such file to its reason."""

    def __init__(self, failed: dict):
        self.failed = failed
        super().__init__('; '.join(f'{k}: {v}' for k, v in failed.items()))


def flac_decode_streams(streams, device, pcm: bool = False) -> list:
    """ttsb_flac_decode_batch on a list of FlacStream in one call -> per stream a dict: 'mono' (float32, what read_wav returns for
    the same PCM as WAV), 'rate', 'pcm' (int32 (total, channels) with pcm=True) and 'error' (None, or the reason and frame index of
    a malformed stream, whose samples are then zeros).  The other streams of the call decode normally."""
    streams = list(streams)
    if not streams:
        return []
    frames = [st.data[st.frame_offset:] for st in streams]
    byte_off = np.concatenate([[0], np.cumsum([len(b) for b in frames])]).astype(np.int64)
    totals = np.array([st.total_samples for st in streams], np.int64)
    widths = totals * np.array([st.channels for st in streams], np.int64)
    dev = torch.device(device)
    with torch.cuda.device(dev):
        blob = np.frombuffer(b''.join(frames), np.uint8)
        data = torch.from_numpy(blob.copy()).to(dev) if len(blob) else torch.empty(0, dtype=torch.uint8, device=dev)
        mono = torch.empty(int(totals.sum()), dtype=torch.float32, device=dev)
        status = torch.empty((len(streams), 2), dtype=torch.int32, device=dev)
        pcm_out = torch.empty(int(widths.sum()), dtype=torch.int32, device=dev) if pcm else None
        lib.flac_decode_batch(data, byte_off, [st.stream_info() for st in streams], mono, status, pcm_out)
        mono, status = mono.cpu().numpy(), status.cpu().numpy()
        pcm_host = pcm_out.cpu().numpy() if pcm else None
    out, mo, po = [], np.concatenate([[0], np.cumsum(totals)]), np.concatenate([[0], np.cumsum(widths)])
    for i, st in enumerate(streams):
        code, frame = int(status[i, 0]), int(status[i, 1])
        err = None if code == 0 else f'{lib.FLAC_STATUS[code]} (frame {frame})'
        out.append(dict(mono=mono[mo[i]:mo[i + 1]], rate=st.sample_rate, error=err,
                        pcm=pcm_host[po[i]:po[i + 1]].reshape(-1, st.channels) if pcm else None))
    return out


def resampled_length(n_samples: int, sr_orig: int, sr_new: int) -> int:
    """Samples of a clip of `n_samples` at sr_orig after resampling to sr_new: ceil(n ratio) in float64, as librosa's fix_length.
    Raises TooShortToResample (a ValueError) when int(n ratio) < 1 (resampy has no output sample to compute)."""
    if sr_orig == sr_new:
        return int(n_samples)
    ratio = float(sr_new) / sr_orig
    if int(n_samples * ratio) < 1:
        raise TooShortToResample(f'{n_samples} samples at {sr_orig} Hz are too short to resample to {sr_new} Hz')
    return int(np.ceil(n_samples * ratio))


def _random_phase(shape, seed):
    """exp(2 pi i u), u uniform from a fresh CPU generator (seeded when `seed` is given) -> complex64 CPU tensor."""
    g = torch.Generator(device='cpu')
    if seed is not None:
        g.manual_seed(seed)
    ph = 2 * np.pi * torch.rand(shape, generator=g, dtype=torch.float64)
    return torch.polar(torch.ones_like(ph), ph).to(torch.complex64)


def _clip_frame_counts(frame_offsets, total_frames: int, min_frames: int = 4) -> np.ndarray:
    """Host check of a packed batch's frame offsets (n_clips + 1, from 0 to total_frames) -> frames per clip.  Griffin-Lim needs
    at least min_frames (Audio.min_griffinlim_frames: 4 at the reference configuration) frames per clip: the STFT of a shorter
    clip's hop (T - 1) samples has no room for the n_fft / 2 samples of reflect padding."""
    off = np.asarray(frame_offsets.cpu() if torch.is_tensor(frame_offsets) else frame_offsets, dtype=np.int64)
    if off.ndim != 1 or len(off) < 2 or off[0] != 0 or off[-1] != total_frames:
        raise ValueError(f'frame offsets must run from 0 to {total_frames} over n_clips + 1 entries, got {off.tolist()}')
    counts = np.diff(off)
    for c, t in enumerate(counts):
        if t < min_frames:
            raise ValueError(f'clip {c} has {t} frames; Griffin-Lim needs at least {min_frames} frames per clip')
    return counts


# the configuration the fused kernels of stft_mel.cu and griffin_lim.cu implement; every other supported one runs through the
# general entry points of stft_general.cu
REFERENCE_STFT = (1024, 256, 1024)
MAX_MEL_CHANNELS = 128


def check_audio_settings(sampling_rate, n_fft, mel_channels, hop_length, win_length, f_min, f_max) -> float:
    """Refuse audio settings outside the supported set, naming the setting and its allowed range -> f_max in Hz (None: sr / 2)."""
    def whole(v):
        return isinstance(v, (int, np.integer)) and not isinstance(v, bool)
    if not whole(sampling_rate) or sampling_rate <= 0:
        raise ValueError(f'sampling_rate must be a positive integer, got {sampling_rate!r}')
    if not whole(n_fft) or not 256 <= n_fft <= 4096 or n_fft & (n_fft - 1):
        raise ValueError(f'n_fft must be a power of two in [256, 4096], got {n_fft!r}')
    # a periodic Hann of one sample is 0.5 - 0.5 cos 0 = 0 (scipy's get_window, which librosa calls, returns [1.0] instead): a
    # window of one sample is refused rather than computed differently from the reference
    if not whole(win_length) or not 2 <= win_length <= n_fft:
        raise ValueError(f'win_length must be an integer in [2, n_fft = {n_fft}], got {win_length!r}')
    if not whole(hop_length) or not 1 <= hop_length <= win_length:
        raise ValueError(f'hop_length must be an integer in [1, win_length = {win_length}], got {hop_length!r}')
    if not whole(mel_channels) or not 1 <= mel_channels <= MAX_MEL_CHANNELS:
        raise ValueError(f'mel_channels must be an integer in [1, {MAX_MEL_CHANNELS}], got {mel_channels!r}')
    nyquist = sampling_rate / 2.0
    fmax = nyquist if f_max is None else f_max
    if not 0 <= f_min < fmax <= nyquist:
        raise ValueError(f'need 0 <= f_min < f_max <= sampling_rate / 2 = {nyquist:g} Hz (f_max None means sampling_rate / 2), got '
                         f'f_min {f_min!r}, f_max {f_max!r}')
    return fmax


class Normalizer:
    code = -1


class MelGAN(Normalizer):
    """log(clip(S, 1e-5)) (reference: data/audio.py:209-216)."""
    code = 0

    def denormalize(self, S):
        return np.exp(S)


class WaveRNN(Normalizer):
    """clip((20 log10(max(1e-5, S)) + 100) / 100, 0, 1) * 8 - 4 (reference: data/audio.py:222-231)."""
    code = 1

    def denormalize(self, S):
        S = (S + 4) / 8
        return np.power(10.0, ((np.clip(S, 0, 1) * 100) - 100) * 0.05)


class Audio:
    def __init__(self, sampling_rate: int, n_fft: int, mel_channels: int, hop_length: int, win_length: int, f_min: int,
                 f_max: int, normalizer: str, device: str = 'cuda:0', **kwargs):
        self.config = dict(sampling_rate=sampling_rate, n_fft=n_fft, mel_channels=mel_channels, hop_length=hop_length,
                           win_length=win_length, f_min=f_min, f_max=f_max, normalizer=normalizer, **kwargs)
        f_max = check_audio_settings(sampling_rate, n_fft, mel_channels, hop_length, win_length, f_min, f_max)
        self._reference_stft = (n_fft, hop_length, win_length) == REFERENCE_STFT
        self.sampling_rate, self.n_fft, self.mel_channels = sampling_rate, n_fft, mel_channels
        self.hop_length, self.win_length, self.f_min, self.f_max = hop_length, win_length, f_min, f_max
        self.normalizer = {'MelGAN': MelGAN, 'WaveRNN': WaveRNN}[normalizer]()
        self.device = torch.device(device)
        self._basis = None
        # the preprocessing settings of the reference's audio section (data/audio.py:24-33); None when absent
        self.norm_wav, self.target_dBFS, self.int16_max = (kwargs.get(k) for k in ('norm_wav', 'target_dBFS', 'int16_max'))
        self.trim_silence, self.trim_long_silences = kwargs.get('trim_silence'), kwargs.get('trim_long_silences')
        self.trim_silence_top_db = kwargs.get('trim_silence_top_db')

    @classmethod
    def from_config(cls, config: dict):
        return cls(**config)

    @property
    def min_mel_samples(self) -> int:
        """Shortest clip the log-mel front end takes: reflect padding needs more than n_fft / 2 samples."""
        return self.n_fft // 2 + 1

    @property
    def min_griffinlim_frames(self) -> int:
        """Fewest frames per clip Griffin-Lim takes: its hop (T - 1) samples must be more than n_fft / 2 (4 at 1024 / 256)."""
        return self.n_fft // 2 // self.hop_length + 2

    def _mel_basis(self) -> torch.Tensor:
        if self._basis is None:
            basis = slaney_mel_basis(self.sampling_rate, self.n_fft, self.mel_channels, self.f_min, self.f_max)
            self._band = mel_band(basis)
            self._basis = torch.from_numpy(basis).to(self.device).contiguous()
        return self._basis

    def _mel_band(self) -> np.ndarray:
        """Band table (n_mels, 2) int32 of the mel basis in host memory, as the fused log-mel kernels take it."""
        self._mel_basis()
        return self._band

    def mel_spectrogram_device(self, wav: torch.Tensor) -> torch.Tensor:
        with torch.cuda.device(self.device):
            return self._mel_spectrogram_device(wav)

    def _mel_spectrogram_device(self, wav: torch.Tensor) -> torch.Tensor:
        """wav fp32 CUDA (n_clips, n_samples) -> fp32 CUDA (n_clips, 1 + n_samples//hop, n_mels)."""
        n_clips, n_samples = wav.shape
        out = torch.empty((n_clips, 1 + n_samples // self.hop_length, self.mel_channels), dtype=torch.float32, device=wav.device)
        if self._reference_stft:
            lib.stft_mel_log(wav.contiguous(), self._mel_basis(), self._mel_band(), self.normalizer.code, out)
        else:
            so = np.arange(n_clips + 1, dtype=np.int64) * n_samples
            fo = np.arange(n_clips + 1, dtype=np.int64) * out.shape[1]
            lib.stft_mel_log_ragged(wav.contiguous().reshape(-1), so, fo, self.n_fft, self.hop_length, self.win_length, self._mel_basis(),
                                    self._inverse_tables()['band'], self.normalizer.code, out)
        return out

    # ---- mel -> waveform (data/audio.py:94-110)
    def _inverse_tables(self):
        """Host-side constants of the mel inversion: pinv(A) (the least-squares start librosa's nnls uses), 1/|A|_2^2, and the
        sparsity pattern of the mel basis (rows are bands, every bin belongs to <= 2 rows)."""
        if getattr(self, '_inv', None) is None:
            A = slaney_mel_basis(self.sampling_rate, self.n_fft, self.mel_channels, self.f_min, self.f_max).astype(np.float64)
            nz = A != 0
            band = mel_band(A)
            bins = np.zeros((A.shape[1], 2), dtype=np.int32)
            for k in range(A.shape[1]):
                idx = np.nonzero(nz[:, k])[0]
                bins[k] = (idx[0], idx[-1] + 1) if len(idx) else (0, 0)
            dev = self.device
            self._inv = dict(pinv=torch.from_numpy(np.linalg.pinv(A).astype(np.float32)).to(dev).contiguous(),
                             step=float(1.0 / np.linalg.norm(A, 2) ** 2), band=torch.from_numpy(band).to(dev).contiguous(),
                             bins=torch.from_numpy(bins).to(dev).contiguous())
        return self._inv

    def mel_to_linear_device(self, mel_amp: torch.Tensor, n_iter: int = 64) -> torch.Tensor:
        """mel amplitudes (T, n_mels) CUDA -> linear magnitudes (T, n_fft/2 + 1) CUDA (librosa mel_to_stft(power=1), see ttsb.h)."""
        with torch.cuda.device(self.device):
            inv = self._inverse_tables()
            out = torch.empty((mel_amp.shape[0], self.n_fft // 2 + 1), dtype=torch.float32, device=self.device)
            to_linear = lib.mel_to_linear if self._reference_stft else lib.mel_to_linear_ex
            to_linear(mel_amp.contiguous(), self._mel_basis(), inv['pinv'], inv['band'], inv['bins'], inv['step'], n_iter, out)
            return out

    def griffinlim_device(self, S: torch.Tensor, n_iter: int = 32, momentum: float = 0.99, init_angles: torch.Tensor = None,
                          seed: int = None) -> torch.Tensor:
        """librosa.griffinlim on the GPU: S (T, n_fft/2 + 1) magnitudes -> waveform (hop (T-1)).  init_angles: unit-modulus
        complex64 (T, n_fft/2 + 1); default: exp(2 pi i u), u uniform (the reference draws it from numpy's global RNG)."""
        if not self._reference_stft:
            return self.griffinlim_batch_device(S, [0, S.shape[0]], n_iter=n_iter, momentum=momentum, init_angles=init_angles,
                                                seeds=[seed])
        with torch.cuda.device(self.device):
            dev = self.device
            T = S.shape[0]
            if init_angles is None:
                init_angles = _random_phase(tuple(S.shape), seed)
            proj = torch.view_as_real((S.to(torch.complex64) * init_angles.to(dev)).contiguous()).contiguous()
            ws = torch.empty(lib.istft_workspace_bytes(T) // 4, dtype=torch.float32, device=dev)
            wav = torch.empty(self.hop_length * (T - 1), dtype=torch.float32, device=dev)
            rebuilt, prev = torch.empty_like(proj), None
            S = S.contiguous()
            for _ in range(n_iter):
                lib.istft(proj, ws, wav)
                spare = prev if prev is not None else torch.empty_like(proj)
                lib.stft_complex(wav, spare)                    # `spare` becomes the new rebuilt spectrum
                lib.griffinlim_update(spare, rebuilt if prev is not None else None, S, momentum, proj)
                prev, rebuilt = rebuilt, spare
            lib.istft(proj, ws, wav)
            return wav

    def reconstruct_waveform(self, mel: np.ndarray, n_iter: int = 32, nnls_iter: int = 64, init_angles=None, seed: int = None) -> np.ndarray:
        """reference: data/audio.py:94-110.  mel: normalised (n_mels, T) as the reference passes it -> waveform float32."""
        m = np.asarray(mel, dtype=np.float32)
        amp = torch.from_numpy(np.ascontiguousarray(self._denormalize(m).T.astype(np.float32))).to(self.device)   # (T, n_mels)
        S = self.mel_to_linear_device(amp, nnls_iter)
        ia = None if init_angles is None else torch.as_tensor(np.ascontiguousarray(np.asarray(init_angles).T)).to(torch.complex64)
        return self.griffinlim_device(S, n_iter=n_iter, init_angles=ia, seed=seed).cpu().numpy()

    def griffinlim_batch_device(self, S: torch.Tensor, frame_offsets, n_iter: int = 32, momentum: float = 0.99,
                                init_angles: torch.Tensor = None, seeds=None) -> torch.Tensor:
        """griffinlim_device for every clip of a packed batch in one pass (ttsb_griffinlim_batch, one launch per stage and
        iteration whatever the number of clips).  S: magnitudes (F, n_fft/2 + 1) on the device, clip c in frames
        frame_offsets[c] .. frame_offsets[c+1] - 1 -> packed waveform (hop (F - n_clips)); clip c starts at sample
        hop (frame_offsets[c] - c).  init_angles: unit-modulus complex64 (F, n_fft/2 + 1); default: clip c draws its phase as
        griffinlim_device(S_c, seed=seeds[c]) does (seeds=None: as griffinlim_device(S_c))."""
        with torch.cuda.device(self.device):
            dev = self.device
            F = S.shape[0]
            counts = _clip_frame_counts(frame_offsets, F, self.min_griffinlim_frames)
            n_clips = len(counts)
            if init_angles is None:
                if seeds is not None and len(seeds) != n_clips:
                    raise ValueError(f'{len(seeds)} seeds for {n_clips} clips')
                init_angles = torch.cat([_random_phase((int(t), S.shape[1]), None if seeds is None else seeds[c])
                                         for c, t in enumerate(counts)])
            init_angles = init_angles.to(device=dev, dtype=torch.complex64).contiguous()
            wav = torch.empty(self.hop_length * (F - n_clips), dtype=torch.float32, device=dev)
            if not self._reference_stft:
                lib.griffinlim_ragged(S.contiguous(), init_angles, np.concatenate([[0], np.cumsum(counts)]), self.n_fft, self.hop_length,
                                      self.win_length, n_iter, momentum, wav)
                return wav
            off = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)).to(dev)
            ws = torch.empty(lib.griffinlim_batch_workspace_bytes(F, n_clips) // 4, dtype=torch.float32, device=dev)
            lib.griffinlim_batch(S.contiguous(), init_angles, off, n_iter, momentum, ws, wav)
            return wav

    def reconstruct_waveform_batch(self, mels, n_iter: int = 32, nnls_iter: int = 64, init_angles=None, seed: int = None) -> list:
        """reconstruct_waveform for a list of normalised mels (n_mels, T_c) in one pass: one mel inversion over the frames of all
        clips, one batched Griffin-Lim -> list of float32 waveforms (hop (T_c - 1)).  With seed=s, clip c gets the phase of
        reconstruct_waveform(mels[c], seed=s + c); init_angles: a list of (n_fft/2 + 1, T_c) arrays, as reconstruct_waveform takes."""
        ms = [np.asarray(m, dtype=np.float32) for m in mels]
        if not ms:
            return []
        for c, m in enumerate(ms):
            if m.ndim != 2 or m.shape[1] < self.min_griffinlim_frames:
                raise ValueError(f'mel {c} has shape {m.shape}; Griffin-Lim needs (n_mels, T) with T >= {self.min_griffinlim_frames} '
                                 f'frames')
        counts = [m.shape[1] for m in ms]
        amp = np.concatenate([self._denormalize(m).T.astype(np.float32) for m in ms])       # (F, n_mels)
        S = self.mel_to_linear_device(torch.from_numpy(np.ascontiguousarray(amp)).to(self.device), nnls_iter)
        ia = None
        if init_angles is not None:
            ia = torch.cat([torch.as_tensor(np.ascontiguousarray(np.asarray(a).T)).to(torch.complex64) for a in init_angles])
        seeds = None if seed is None else [seed + c for c in range(len(ms))]
        off = np.concatenate([[0], np.cumsum(counts)])
        wav = self.griffinlim_batch_device(S, off, n_iter=n_iter, init_angles=ia, seeds=seeds).cpu().numpy()
        starts = self.hop_length * (off[:-1] - np.arange(len(ms)))
        return [wav[s:s + self.hop_length * (t - 1)] for s, t in zip(starts, counts)]

    def save_wav(self, y: np.ndarray, wav_path):
        """reference: data/audio.py:143-144 (soundfile.write(wav_path, y, sampling_rate): 16-bit PCM for .wav).  Samples are
        scaled by 32767 and rounded to nearest as libsndfile does; samples beyond full scale are clipped to the int16 range
        (libsndfile, without its clipping option, wraps them around)."""
        import wave
        x = np.asarray(y, dtype=np.float32).reshape(-1)
        pcm = np.clip(np.rint(x * np.float32(32767)), -32768, 32767).astype('<i2')
        with wave.open(str(wav_path), 'wb') as f:
            f.setnchannels(1)
            f.setsampwidth(2)
            f.setframerate(int(self.sampling_rate))
            f.writeframes(pcm.tobytes())

    def _denormalize(self, S):
        return self.normalizer.denormalize(S)

    def mel_spectrogram_batch(self, wavs: np.ndarray) -> np.ndarray:
        w = torch.from_numpy(np.ascontiguousarray(wavs, dtype=np.float32)).to(self.device)
        return self.mel_spectrogram_device(w).cpu().numpy()

    def mel_spectrogram(self, wav: np.ndarray) -> np.ndarray:
        """This is what the model is trained to reproduce (reference: data/audio.py:88-92) -> (T, n_mels) float32."""
        return self.mel_spectrogram_batch(np.asarray(wav, dtype=np.float32)[None])[0]

    def _frames_per_clip(self, lengths) -> np.ndarray:
        return np.array([1 + int(L) // self.hop_length for L in lengths], dtype=np.int64)

    def _pitch_frames(self, lengths) -> np.ndarray:
        """WORLD's frame count int(1000 L / fs / frame_period) + 1 at the reference's frame period hop / fs * 1000 ms."""
        fp = self.hop_length / self.sampling_rate * 1000
        return np.array([int(1000.0 * int(L) / self.sampling_rate / fp) + 1 for L in lengths], dtype=np.int64)

    def _pack(self, wavs):
        """list of 1-D waveforms -> (packed fp32 device tensor, sample offsets (n + 1) int64)."""
        ws = [np.asarray(w, dtype=np.float32).reshape(-1) for w in wavs]
        if not ws:
            raise ValueError('no clips')
        so = np.concatenate([[0], np.cumsum([len(w) for w in ws])]).astype(np.int64)
        return torch.from_numpy(np.concatenate(ws)).to(self.device), so

    def mel_spectrogram_ragged_device(self, wav: torch.Tensor, sample_offsets) -> tuple:
        """ttsb_stft_mel_log_batch (ttsb_stft_mel_log_ragged away from the reference configuration): packed fp32 clips on the
        device -> (packed log-mels (F, n_mels) on the device, frame offsets).  Clip c's mel is bit-identical to
        mel_spectrogram_device on that clip alone."""
        with torch.cuda.device(self.device):
            so = np.asarray(sample_offsets, dtype=np.int64)
            fo = np.concatenate([[0], np.cumsum(self._frames_per_clip(np.diff(so)))])
            out = torch.empty((int(fo[-1]), self.mel_channels), dtype=torch.float32, device=self.device)
            if self._reference_stft:
                lib.stft_mel_log_batch(wav.contiguous(), so, fo, self._mel_basis(), self._mel_band(), self.normalizer.code, out)
            else:
                lib.stft_mel_log_ragged(wav.contiguous(), so, fo, self.n_fft, self.hop_length, self.win_length, self._mel_basis(),
                                        self._inverse_tables()['band'], self.normalizer.code, out)
            return out, fo

    def extract_pitch_device(self, wav: torch.Tensor, sample_offsets, workspace: torch.Tensor = None) -> tuple:
        """ttsb_pitch_dio_stonemask: packed fp32 clips on the device -> (packed float64 f0 on the device, frame offsets).
        `workspace`: a uint8 device tensor to use when it is large enough (the kernels' intermediate results stay in it)."""
        with torch.cuda.device(self.device):
            so = np.asarray(sample_offsets, dtype=np.int64)
            fo = np.concatenate([[0], np.cumsum(self._pitch_frames(np.diff(so)))])
            fp = self.hop_length / self.sampling_rate * 1000
            nb = lib.pitch_workspace_bytes(so, self.sampling_rate, fp)
            if workspace is None or workspace.numel() < nb:
                workspace = torch.empty(nb, dtype=torch.uint8, device=self.device)
            f0 = torch.empty(int(fo[-1]), dtype=torch.float64, device=self.device)
            lib.pitch_dio_stonemask(wav.contiguous(), so, self.sampling_rate, fp, fo, f0, workspace)
            return f0, fo

    def extract_pitch_batch(self, wavs) -> list:
        """extract_pitch of every clip of a list in one pass -> list of float64 (T_c,)."""
        wav, so = self._pack(wavs)
        f0, fo = self.extract_pitch_device(wav, so)
        f0 = f0.cpu().numpy()
        return [f0[a:b] for a, b in zip(fo[:-1], fo[1:])]

    def extract_pitch(self, y: np.ndarray) -> np.ndarray:
        """reference: data/audio.py:146-151 (pw.dio(y, fs, frame_period=hop/fs*1000) then pw.stonemask) -> float64 (T,)."""
        return self.extract_pitch_batch([y])[0]

    @property
    def cheaptrick_fft_size(self) -> int:
        """pyworld's CheapTrick FFT size at f0_floor 71 Hz: 2^(1 + int(log2(3 fs / 71 + 1))) (1024 at 16 to 24 kHz, 2048 at 44.1
        and 48 kHz)."""
        return 1 << (1 + int(np.log(3.0 * self.sampling_rate / 71.0 + 1) / np.log(2.0)))

    def spectral_envelope_device(self, wav: torch.Tensor, sample_offsets, f0: torch.Tensor, f0_offsets) -> tuple:
        """ttsb_cheaptrick (pyworld.cheaptrick with q1 -0.15, f0_floor 71): packed fp32 clips and their float64 F0 at WORLD's frames
        (extract_pitch_device) on the device -> (packed float64 envelopes (frames, cheaptrick_fft_size / 2 + 1) on the device, frame
        offsets).  Clip c's envelope does not depend on the other clips."""
        with torch.cuda.device(self.device):
            so = np.asarray(sample_offsets, dtype=np.int64)
            fo = np.asarray(f0_offsets, dtype=np.int64)
            n = self.cheaptrick_fft_size
            env = torch.empty((int(fo[-1]), n // 2 + 1), dtype=torch.float64, device=self.device)
            fp = self.hop_length / self.sampling_rate * 1000
            lib.cheaptrick(wav.contiguous(), so, self.sampling_rate, fp, f0.contiguous(), fo, -0.15, n, env)
            return env, fo

    def world_mcep_batch(self, wavs, order: int = 24, alpha: float = None) -> list:
        """WORLD mel-cepstra of every clip of a list: DIO + StoneMask (extract_pitch_device), CheapTrick (spectral_envelope_device)
        and pysptk's sp2mc (ttsb_sp2mc) on one packed upload per PITCH_CHUNK_SAMPLES samples, at the frame period of the training
        data -> list of float64 (T_c, order + 1).  alpha None: mcep_alpha(sampling_rate).  A clip too short for DIO raises
        ValueError."""
        from ..utils.evaluation import PITCH_CHUNK_SAMPLES, _dio_takes, mcep_alpha, sp2mc_matrix
        ws = [np.asarray(w, dtype=np.float32).reshape(-1) for w in wavs]
        for c, w in enumerate(ws):
            if not _dio_takes(self, len(w)):
                raise ValueError(f'clip {c} has {len(w)} samples; DIO needs more WORLD frames than its voice_range_minimum')
        alpha = mcep_alpha(self.sampling_rate) if alpha is None else float(alpha)
        n = self.cheaptrick_fft_size
        key = (n, int(order), alpha)
        if getattr(self, '_sp2mc', (None,))[0] != key:
            self._sp2mc = (key, torch.from_numpy(sp2mc_matrix(n, int(order), alpha)).to(self.device).contiguous())
        W = self._sp2mc[1]
        chunks, samples = [[]], 0
        for c, w in enumerate(ws):
            if chunks[-1] and samples + len(w) > PITCH_CHUNK_SAMPLES:
                chunks.append([])
                samples = 0
            chunks[-1].append(c)
            samples += len(w)
        out = [None] * len(ws)
        with torch.cuda.device(self.device):
            for chunk in chunks:
                if not chunk:
                    continue
                wav, so = self._pack([ws[c] for c in chunk])
                f0, fo = self.extract_pitch_device(wav, so)
                env, _ = self.spectral_envelope_device(wav, so, f0, fo)
                mc = torch.empty((env.shape[0], int(order) + 1), dtype=torch.float64, device=self.device)
                lib.sp2mc(env, W, mc)
                mc = mc.cpu().numpy()
                for r, c in enumerate(chunk):
                    out[c] = mc[fo[r]:fo[r + 1]]
        return out

    def mel_spectrogram_ragged(self, wavs) -> list:
        """mel_spectrogram of every clip of a list in one launch -> list of (T_c, n_mels) float32, T_c = 1 + L_c // hop."""
        wav, so = self._pack(wavs)
        mel, fo = self.mel_spectrogram_ragged_device(wav, so)
        mel = mel.cpu().numpy()
        return [mel[a:b] for a, b in zip(fo[:-1], fo[1:])]

    def _resample_window(self) -> torch.Tensor:
        if getattr(self, '_rs_window', None) is None:
            self._rs_window = torch.from_numpy(kaiser_best_half_window()).to(self.device).contiguous()
        return self._rs_window

    def resample_ragged_device(self, wav: torch.Tensor, sample_offsets, src_rates) -> tuple:
        """ttsb_resample_batch: packed fp32 clips on the device, clip c sampled at src_rates[c] Hz -> (packed fp32 clips at
        sampling_rate on the device, output sample offsets).  What librosa.load(sr=sampling_rate) does after reading and mixing to
        mono (resampy kaiser_best, then fix_length to ceil(L ratio)); a clip already at sampling_rate comes back unchanged.  Clip
        c's output does not depend on the other clips.  A clip too short to resample raises ValueError."""
        with torch.cuda.device(self.device):
            so = np.asarray(sample_offsets, dtype=np.int64)
            rates = np.asarray(src_rates, dtype=np.int64).reshape(-1)
            if len(rates) != len(so) - 1:
                raise ValueError(f'{len(rates)} source rates for {len(so) - 1} clips')
            lengths = []
            for c, (L, sr) in enumerate(zip(np.diff(so), rates)):
                try:
                    lengths.append(resampled_length(int(L), int(sr), self.sampling_rate))
                except ValueError as e:
                    raise ValueError(f'clip {c}: {e}') from None
            oo = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
            out = torch.empty(int(oo[-1]), dtype=torch.float32, device=self.device)
            lib.resample_batch(wav.contiguous(), so, rates, self.sampling_rate, self._resample_window(), oo, out)
            return out, oo

    def resample_ragged(self, clips) -> list:
        """resample_ragged_device for a list of (float32 samples, rate) in one launch -> list of float32 arrays at sampling_rate."""
        clips = list(clips)
        wav, so = self._pack([y for y, _ in clips])
        out, oo = self.resample_ragged_device(wav, so, [sr for _, sr in clips])
        out = out.cpu().numpy()
        return [out[a:b] for a, b in zip(oo[:-1], oo[1:])]

    def trim_silence_bounds_device(self, wav: torch.Tensor, sample_offsets) -> torch.Tensor:
        """ttsb_trim_silence_bounds at trim_silence_top_db: packed fp32 clips on the device -> int32 (n_clips, 2) on the device,
        [start, end) of each clip's samples that librosa.effects.trim(y, top_db, frame_length=256, hop_length=64) keeps,
        relative to the clip.  Clip c's bounds do not depend on the other clips."""
        top_db = self._trim_top_db()
        with torch.cuda.device(self.device):
            so = np.asarray(sample_offsets, dtype=np.int64)
            bounds = torch.empty((len(so) - 1, 2), dtype=torch.int32, device=self.device)
            lib.trim_silence_bounds(wav.contiguous(), so, top_db, bounds)
            return bounds

    def trim_silence_ragged(self, wavs) -> list:
        """trim_audio_silence of every clip of a list in one launch -> list of float32 arrays (slices of the float32 clips)."""
        self._trim_top_db()             # refuse a missing setting before anything reaches the device
        ws = [np.asarray(w, dtype=np.float32).reshape(-1) for w in wavs]
        wav, so = self._pack(ws)
        bounds = self.trim_silence_bounds_device(wav, so).cpu().numpy()
        return [w[a:b] for w, (a, b) in zip(ws, bounds)]

    def trim_audio_silence(self, wav) -> np.ndarray:
        """reference: data/audio.py:164-169 (librosa.effects.trim(wav, top_db=trim_silence_top_db, frame_length=256,
        hop_length=64)[0])."""
        return self.trim_silence_ragged([wav])[0]

    def _trim_top_db(self) -> float:
        if self.trim_silence_top_db is None:
            raise NotImplementedError('trim_silence needs librosa.effects.trim\'s top_db, and the audio settings have no '
                                      'trim_silence_top_db; set it (the reference uses 60) or set trim_silence: false')
        return float(self.trim_silence_top_db)

    def read_wav(self, wav_path):
        """The decoding half of librosa.load (data/audio.py:126-130) -> (float32 mono samples, the file's own rate).  PCM and float
        WAV, several channels averaged to mono; PCM is scaled as libsndfile reads it into float (int16 / 32768, ...)."""
        from scipy.io import wavfile
        sr, data = wavfile.read(str(wav_path))
        if data.dtype == np.uint8:
            y = (data.astype(np.float32) - np.float32(128)) / np.float32(128)
        elif data.dtype.kind == 'i':
            y = data.astype(np.float32) / np.float32(2 ** (8 * data.dtype.itemsize - 1))
        else:
            y = data.astype(np.float32)
        if y.ndim == 2:
            y = np.mean(y, axis=1)
        return y, sr

    def read_flac_batch(self, paths) -> list:
        """The decoding half of librosa.load for .flac files (data/audio.py:126-130; libsndfile reads FLAC) -> list of (float32 mono
        samples, the file's own rate), all files decoded in one ttsb_flac_decode_batch call.  The samples equal read_wav's of the
        same PCM stored as WAV, bit for bit.  Malformed metadata raises ValueError naming the file; malformed frames raise
        FlacDecodeError naming every failed file, its reason and frame."""
        streams = [p if isinstance(p, FlacStream) else FlacStream.read(p) for p in paths]
        res = flac_decode_streams(streams, self.device)
        failed = {st.path: r['error'] for st, r in zip(streams, res) if r['error']}
        if failed:
            raise FlacDecodeError(failed)
        return [(r['mono'], r['rate']) for r in res]

    def read_audio(self, path):
        """read_wav, or read_flac_batch for a .flac file -> (float32 mono samples, the file's own rate)."""
        if str(path).lower().endswith('.flac'):
            return self.read_flac_batch([path])[0]
        return self.read_wav(path)

    def read_for_batch(self, wav_path):
        """The per-file half of preparing a recording as create_training_data.py does (load_wavs): -> (samples, None), read and
        preprocessed up to the trim (all of preprocess without trim_silence), when the file is at sampling_rate; else (the raw mono
        samples, the file's rate) for finish_batch to resample.  A .flac file is returned undecoded, as (FlacStream, None), for
        finish_batch to decode with the rest of the batch.  A file too short to resample raises TooShortToResample."""
        if str(wav_path).lower().endswith('.flac'):
            st = FlacStream.read(wav_path)
            resampled_length(st.total_samples, st.sample_rate, self.sampling_rate)
            return st, None
        y, sr = self.read_wav(wav_path)
        if sr == self.sampling_rate:
            return self._host_preprocess()(y), None
        resampled_length(len(y), sr, self.sampling_rate)
        return y, sr

    def finish_batch(self, items) -> list:
        """The batch half of load_wavs on read_for_batch items: the FLAC files decoded in one call (read_flac_batch), after which
        each takes the path of a WAV file's samples at its rate; the off-rate clips resampled in one launch (resample_ragged) and
        preprocessed; with trim_silence, every clip trimmed in one launch (trim_silence_ragged) and padded to the hop -> list of
        float32 arrays at sampling_rate, each what preprocess makes of the file's samples at that rate."""
        items = list(items)
        flac = [c for c, (y, _) in enumerate(items) if isinstance(y, FlacStream)]
        if flac:
            preprocess = self._host_preprocess()
            for c, (y, sr) in zip(flac, self.read_flac_batch([items[c][0] for c in flac])):
                items[c] = (preprocess(y), None) if sr == self.sampling_rate else (y, sr)
        off = [c for c, (_, sr) in enumerate(items) if sr is not None]
        done = dict(zip(off, self.resample_ragged([items[c] for c in off]))) if off else {}
        preprocess = self._host_preprocess()
        clips = [preprocess(done[c]) if c in done else y for c, (y, _) in enumerate(items)]
        if self.trim_silence:
            clips = [self.pad_to_hop(y) for y in self.trim_silence_ragged(clips)]
        return clips

    def load_wavs(self, wav_paths) -> list:
        """Recordings as create_training_data.py prepares them before their mels: read_wav or the GPU FLAC decoder (one call for
        all .flac files), GPU resampling of an off-rate file,
        volume normalisation, trim_silence when configured, the pad to the hop -> list of float32 arrays."""
        return self.finish_batch([self.read_for_batch(p) for p in wav_paths])

    def _host_preprocess(self):
        """The part of preprocess done per file: all of it, or with trim_silence everything before the trim (the trim and the hop
        padding run a batch at a time in finish_batch)."""
        return self.preprocess_before_trim if self.trim_silence else self.preprocess

    def load_wav(self, wav_path, preprocess: bool = True):
        """reference: data/audio.py:126-130 (librosa.load(path, sr=sampling_rate)) -> (float32 samples, rate): read_wav (or
        read_flac_batch for a .flac file), then preprocess.  A file at another rate is refused here; read it with read_audio and
        resample it with resample_ragged (what create_training_data.py does for a whole corpus)."""
        y, sr = self.read_audio(wav_path)
        if sr != self.sampling_rate:
            raise ValueError(f'{wav_path}: sampled at {sr} Hz, expected {self.sampling_rate} Hz; read_wav + resample_ragged '
                             f'resample it')
        if preprocess:
            y = self.preprocess(y)
        return y, sr

    def preprocess(self, y):
        """reference: data/audio.py:132-141.  trim_long_silences is refused; trim_silence runs on the GPU (trim_audio_silence)."""
        y = self.preprocess_before_trim(y)
        if self.trim_silence:
            y = self.trim_audio_silence(y)
        return self.pad_to_hop(y)

    def preprocess_before_trim(self, y):
        """The host part of preprocess before the silence trim: volume normalisation, and the refusal of the trims this project
        does not implement (trim_long_silences; trim_silence without trim_silence_top_db)."""
        if self.norm_wav:
            y = self.normalize_volume(y, increase_only=True)
        if self.trim_long_silences:
            raise NotImplementedError('trim_long_silences needs webrtcvad voice-activity detection, which this project does not '
                                      'implement; set trim_long_silences: false in the audio settings')
        if self.trim_silence:
            self._trim_top_db()
        return y

    def pad_to_hop(self, y):
        """The last step of preprocess: one zero sample appended to a clip whose length is a multiple of hop_length."""
        if y.shape[0] % self.hop_length == 0:
            y = np.pad(y, (0, 1))
        return y

    def normalize_volume(self, wav, increase_only=False, decrease_only=False):
        """reference: data/audio.py:154-162, the same expressions."""
        if increase_only and decrease_only:
            raise ValueError("Both increase only and decrease only are set")
        rms = np.sqrt(np.mean((wav * self.int16_max) ** 2))
        wave_dBFS = 20 * np.log10(rms / self.int16_max)
        dBFS_change = self.target_dBFS - wave_dBFS
        if dBFS_change < 0 and increase_only or dBFS_change > 0 and decrease_only:
            return wav
        return wav * (10 ** (dBFS_change / 20))
