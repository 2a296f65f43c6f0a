"""Log-mel front end with the reference's ``FeatureExtractor`` interface, computed on the GPU.

Mirrors ``faster_whisper/feature_extractor.py:4-230`` (constructor arguments, attributes, ``__call__``
semantics including the ``chunk_length`` side effect at ``:203-205``).  ``__call__`` hands the waveform to the
fused CUDA kernel through the C ABI (``b2w_logmel``); there is no NumPy fallback — without the CUDA library
and an H100 the call raises.
"""

from __future__ import annotations

import numpy as np

from . import engine


class FeatureExtractor:
    def __init__(self, feature_size=80, sampling_rate=16000, hop_length=160, chunk_length=30, n_fft=400, device_index=0):
        if (sampling_rate, hop_length, n_fft) != (16000, 160, 400):
            raise ValueError("the CUDA log-mel kernel is specialised for Whisper's 16 kHz / n_fft=400 / hop=160 front end")
        if not 1 <= int(feature_size) <= 128:
            raise ValueError("feature_size must be in 1..128")
        self.n_fft = n_fft
        self.hop_length = hop_length
        self.chunk_length = chunk_length
        self.sampling_rate = sampling_rate
        self.n_samples = chunk_length * sampling_rate
        self.nb_max_frames = self.n_samples // hop_length
        self.time_per_frame = hop_length / sampling_rate
        self.feature_size = int(feature_size)
        self.device_index = device_index
        self.mel_filters = self.get_mel_filters(sampling_rate, n_fft, n_mels=feature_size).astype("float32")

    @staticmethod
    def get_mel_filters(sr, n_fft, n_mels=128):
        """Slaney-normalised triangular mel filterbank [n_mels, 1 + n_fft//2] (float64).  The device kernel
        builds the same table in C++ (csrc/mel.cu:build_filters); this copy is the inspectable attribute the
        reference exposes."""
        n_mels = int(n_mels)
        bin_hz = np.fft.rfftfreq(n=n_fft, d=1.0 / sr)
        mel_pts = np.linspace(0.0, 45.245640471924965, n_mels + 2)
        hz = (200.0 / 3) * mel_pts
        knee_hz, knee_mel = 1000.0, 1000.0 / (200.0 / 3)
        upper = mel_pts >= knee_mel
        hz[upper] = knee_hz * np.exp((np.log(6.4) / 27.0) * (mel_pts[upper] - knee_mel))
        width = np.diff(hz)
        dist = hz[:, None] - bin_hz[None, :]
        rising = -dist[:-2] / width[:-1, None]
        falling = dist[2:] / width[1:, None]
        bank = np.clip(np.minimum(rising, falling), 0.0, None)
        return bank * (2.0 / (hz[2:] - hz[:-2]))[:, None]

    def __call__(self, waveform: np.ndarray, padding=160, chunk_length=None):
        """float32 [feature_size, 1 + len(waveform)//160] for the default padding of 160 samples."""
        if chunk_length is not None:
            self.n_samples = chunk_length * self.sampling_rate
            self.nb_max_frames = self.n_samples // self.hop_length
        waveform = np.asarray(waveform)
        if waveform.ndim != 1:
            raise ValueError("expected a mono waveform (1-D array)")
        return engine.log_mel(waveform.astype(np.float32, copy=False), self.feature_size, int(padding or 0), self.device_index)
