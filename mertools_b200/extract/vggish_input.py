"""Log-mel examples of the reference's VGGish audio path, computed on the GPU.

Mirrors MERBench/feature_extraction/audio/vggish/vggish_input.py (``waveform_to_examples`` :37-82,
``wavfile_to_examples`` :85-105) on top of ``mer_logmel`` (mel_features.log_mel_spectrogram with the
constants of vggish_params.py).  Input audio must already be 16 kHz (the reference resamples other rates
with resampy; every MER corpus is extracted at 16 kHz, extract_vggish_embedding.py).  The VGGish network
that consumes these examples is outside the H100 path (SURVEY.md §8f N3/N4).
"""
from __future__ import annotations

import ctypes as C
import math

import numpy as np
import torch

from .. import _lib as L

SAMPLE_RATE = 16000
NUM_FRAMES, NUM_BANDS = 96, 64
STFT_HOP_LENGTH_SECONDS = 0.010
EXAMPLE_WINDOW_SECONDS = 0.96


def log_mel_spectrogram(waves: torch.Tensor) -> torch.Tensor:
    """waves: fp32 CUDA [B, L] at 16 kHz -> [B, num_frames, 64] (mel_features.py:166-223)."""
    assert waves.is_cuda and waves.dtype == torch.float32 and waves.dim() == 2
    waves = waves.contiguous()
    lib = L.lib()
    fn = L.declare("mer_logmel", [C.c_void_p, C.c_int, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p])
    lib.mer_logmel_num_frames.argtypes = [C.c_int]
    B, n = waves.shape
    nf = lib.mer_logmel_num_frames(n)
    assert nf > 0, f"{n} samples are shorter than one 25 ms analysis window"
    out = torch.empty(B, nf, NUM_BANDS, dtype=torch.float32, device=waves.device)
    L.check(fn(L.ptr(waves), B, n, n, L.ptr(out), L.stream_ptr()))
    return out


def frame(data: np.ndarray, window_length: int, hop_length: int) -> np.ndarray:
    """mel_features.frame (:21-45): complete frames only, as a strided view."""
    num_samples = data.shape[0]
    num_frames = 1 + int(np.floor((num_samples - window_length) / hop_length))
    shape = (num_frames, window_length) + data.shape[1:]
    strides = (data.strides[0] * hop_length,) + data.strides
    return np.lib.stride_tricks.as_strided(data, shape=shape, strides=strides)


def waveform_to_examples(data, sample_rate, hop_sec, device="cuda"):
    """[num_examples, 96, 64] log-mel patches of one waveform (vggish_input.py:37-82)."""
    data = np.asarray(data)
    if len(data.shape) > 1:
        data = np.mean(data, axis=1)
    assert sample_rate == SAMPLE_RATE, "mertools_b200 expects 16 kHz audio (the reference resamples with resampy)"
    wave = torch.from_numpy(np.ascontiguousarray(data, dtype=np.float32))[None].to(device)
    log_mel = log_mel_spectrogram(wave)[0].cpu().numpy()
    features_sample_rate = 1.0 / STFT_HOP_LENGTH_SECONDS
    example_window_length = int(round(EXAMPLE_WINDOW_SECONDS * features_sample_rate))
    example_hop_length = int(round(hop_sec * features_sample_rate))
    return frame(log_mel, window_length=example_window_length, hop_length=example_hop_length)


def wavfile_to_examples(wav_file, hop_sec, device="cuda"):
    """vggish_input.py:85-105: int16 PCM -> [-1, 1); clips shorter than one second are tiled."""
    import soundfile as sf
    wav_data, sr = sf.read(wav_file, dtype="int16")
    assert wav_data.dtype == np.int16, "Bad sample type: %r" % wav_data.dtype
    samples = wav_data / 32768.0
    if len(samples) < sr:
        samples = np.array(samples.tolist() * math.ceil(sr / len(samples)))
    return waveform_to_examples(samples, sr, hop_sec, device=device)
