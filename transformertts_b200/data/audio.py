"""Audio front-end mirror of the reference's ``data/audio.py`` for the hot path only: STFT -> 80-bin mel -> log
normalisation (reference: data/audio.py:72-92, 196-231), executed by the fused CUDA kernel ``ttsb_stft_mel_log``.

File I/O, VAD trimming, pitch extraction and Griffin-Lim are outside the hot path (SURVEY.md section 8f).
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
    reference reaches through librosa.feature.melspectrogram at data/audio.py:73-79) -> float32 (n_mels, 1+n_fft/2)."""
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


def _random_phase(shape, seed):
    """exp(2 pi i u), u uniform from a fresh CPU generator (seeded when `seed` is given) -> complex64 CPU tensor."""
    g = torch.Generator(device='cpu')
    if seed is not None:
        g.manual_seed(seed)
    ph = 2 * np.pi * torch.rand(shape, generator=g, dtype=torch.float64)
    return torch.polar(torch.ones_like(ph), ph).to(torch.complex64)


def _clip_frame_counts(frame_offsets, total_frames: int) -> np.ndarray:
    """Host check of a packed batch's frame offsets (n_clips + 1, from 0 to total_frames) -> frames per clip.  Griffin-Lim needs
    at least 4 frames per clip: the STFT of a shorter clip's 256 (T - 1) samples has no room for the 512-sample reflect padding."""
    off = np.asarray(frame_offsets.cpu() if torch.is_tensor(frame_offsets) else frame_offsets, dtype=np.int64)
    if off.ndim != 1 or len(off) < 2 or off[0] != 0 or off[-1] != total_frames:
        raise ValueError(f'frame offsets must run from 0 to {total_frames} over n_clips + 1 entries, got {off.tolist()}')
    counts = np.diff(off)
    for c, t in enumerate(counts):
        if t < 4:
            raise ValueError(f'clip {c} has {t} frames; Griffin-Lim needs at least 4 frames per clip')
    return counts


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
        if (n_fft, hop_length, win_length) != (1024, 256, 1024):
            raise lib.TtsbError('the fused STFT kernel implements the reference configuration n_fft=1024, hop=256, win=1024')
        self.sampling_rate, self.n_fft, self.mel_channels = sampling_rate, n_fft, mel_channels
        self.hop_length, self.win_length, self.f_min, self.f_max = hop_length, win_length, f_min, f_max
        self.normalizer = {'MelGAN': MelGAN, 'WaveRNN': WaveRNN}[normalizer]()
        self.device = torch.device(device)
        self._basis = None

    @classmethod
    def from_config(cls, config: dict):
        return cls(**config)

    def _mel_basis(self) -> torch.Tensor:
        if self._basis is None:
            self._basis = torch.from_numpy(slaney_mel_basis(self.sampling_rate, self.n_fft, self.mel_channels, self.f_min,
                                                            self.f_max)).to(self.device).contiguous()
        return self._basis

    def mel_spectrogram_device(self, wav: torch.Tensor) -> torch.Tensor:
        with torch.cuda.device(self.device):
            return self._mel_spectrogram_device(wav)

    def _mel_spectrogram_device(self, wav: torch.Tensor) -> torch.Tensor:
        """wav fp32 CUDA (n_clips, n_samples) -> fp32 CUDA (n_clips, 1 + n_samples//hop, n_mels)."""
        n_clips, n_samples = wav.shape
        out = torch.empty((n_clips, 1 + n_samples // self.hop_length, self.mel_channels), dtype=torch.float32, device=wav.device)
        lib.stft_mel_log(wav.contiguous(), self._mel_basis(), self.normalizer.code, out)
        return out

    # ---- mel -> waveform (data/audio.py:94-110)
    def _inverse_tables(self):
        """Host-side constants of the mel inversion: pinv(A) (the least-squares start librosa's nnls uses), 1/|A|_2^2, and the
        sparsity pattern of the mel basis (rows are bands, every bin belongs to <= 2 rows)."""
        if getattr(self, '_inv', None) is None:
            A = slaney_mel_basis(self.sampling_rate, self.n_fft, self.mel_channels, self.f_min, self.f_max).astype(np.float64)
            nz = A != 0
            band = np.zeros((A.shape[0], 2), dtype=np.int32)
            for j in range(A.shape[0]):
                idx = np.nonzero(nz[j])[0]
                band[j] = (idx[0], idx[-1] + 1) if len(idx) else (0, 0)
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
        """mel amplitudes (T, n_mels) CUDA -> linear magnitudes (T, 513) CUDA (librosa mel_to_stft(power=1), see ttsb.h)."""
        with torch.cuda.device(self.device):
            inv = self._inverse_tables()
            out = torch.empty((mel_amp.shape[0], self.n_fft // 2 + 1), dtype=torch.float32, device=self.device)
            lib.mel_to_linear(mel_amp.contiguous(), self._mel_basis(), inv['pinv'], inv['band'], inv['bins'], inv['step'], n_iter, out)
            return out

    def griffinlim_device(self, S: torch.Tensor, n_iter: int = 32, momentum: float = 0.99, init_angles: torch.Tensor = None,
                          seed: int = None) -> torch.Tensor:
        """librosa.griffinlim on the GPU: S (T, 513) magnitudes -> waveform (256 (T-1)).  init_angles: unit-modulus complex64
        (T, 513); default: exp(2 pi i u), u uniform (the reference draws it from numpy's global RNG)."""
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
        iteration whatever the number of clips).  S: magnitudes (F, 513) on the device, clip c in frames
        frame_offsets[c] .. frame_offsets[c+1] - 1 -> packed waveform (256 (F - n_clips)); clip c starts at sample
        256 (frame_offsets[c] - c).  init_angles: unit-modulus complex64 (F, 513); default: clip c draws its phase as
        griffinlim_device(S_c, seed=seeds[c]) does (seeds=None: as griffinlim_device(S_c))."""
        with torch.cuda.device(self.device):
            dev = self.device
            F = S.shape[0]
            counts = _clip_frame_counts(frame_offsets, F)
            n_clips = len(counts)
            if init_angles is None:
                if seeds is not None and len(seeds) != n_clips:
                    raise ValueError(f'{len(seeds)} seeds for {n_clips} clips')
                init_angles = torch.cat([_random_phase((int(t), S.shape[1]), None if seeds is None else seeds[c])
                                         for c, t in enumerate(counts)])
            init_angles = init_angles.to(device=dev, dtype=torch.complex64).contiguous()
            off = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)).to(dev)
            ws = torch.empty(lib.griffinlim_batch_workspace_bytes(F, n_clips) // 4, dtype=torch.float32, device=dev)
            wav = torch.empty(self.hop_length * (F - n_clips), dtype=torch.float32, device=dev)
            lib.griffinlim_batch(S.contiguous(), init_angles, off, n_iter, momentum, ws, wav)
            return wav

    def reconstruct_waveform_batch(self, mels, n_iter: int = 32, nnls_iter: int = 64, init_angles=None, seed: int = None) -> list:
        """reconstruct_waveform for a list of normalised mels (n_mels, T_c) in one pass: one mel inversion over the frames of all
        clips, one batched Griffin-Lim -> list of float32 waveforms (256 (T_c - 1)).  With seed=s, clip c gets the phase of
        reconstruct_waveform(mels[c], seed=s + c); init_angles: a list of (513, T_c) arrays, as reconstruct_waveform takes."""
        ms = [np.asarray(m, dtype=np.float32) for m in mels]
        if not ms:
            return []
        for c, m in enumerate(ms):
            if m.ndim != 2 or m.shape[1] < 4:
                raise ValueError(f'mel {c} has shape {m.shape}; Griffin-Lim needs (n_mels, T) with T >= 4 frames')
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
