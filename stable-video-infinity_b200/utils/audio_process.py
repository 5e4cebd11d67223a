"""Host-side audio helpers of SVI-Talk (reference utils/audio_process.py:10-75), with the reference's names.

The reference reads audio with librosa (soundfile + soxr resampling) and normalises loudness with pyloudnorm.  Here:

  * ``audio_prepare_single`` reads WAV files with scipy.io.wavfile (PCM 8/16/24/32-bit, IEEE float), mixes to mono by the
    channel mean and resamples with scipy.signal.resample_poly to librosa's length, ceil(n * 16000 / sr).  Other
    containers (mp3, m4a, flac, video) need ffmpeg or audioread and are refused with a clear error.  resample_poly is not
    soxr: the features of non-16 kHz input differ from the reference's by an amount that has not been measured.
  * ``loudness_norm`` is ITU-R BS.1770 integrated loudness as pyloudnorm's default meter computes it (K-weighting,
    400 ms blocks with 75 % overlap, -70 LUFS absolute and -10 LU relative gates) and the gain to -23 LUFS.
  * ``get_embedding`` runs the wav2vec2 extractor on the GPU (diffsynth.models.wav2vec2) and returns [T, 12, 768].
"""
import math
import os

import numpy as np
import torch

_WAV_EXT = (".wav", ".wave")


def read_wav(path):
    """(float32 samples [n] or [n, channels] scaled to [-1, 1) as soundfile does, sample rate)."""
    from scipy.io import wavfile
    sr, data = wavfile.read(path)
    if data.dtype == np.uint8:
        x = (data.astype(np.float32) - 128.0) / 128.0
    elif data.dtype == np.int16:
        x = data.astype(np.float32) / 32768.0
    elif data.dtype == np.int32:                  # 32-bit PCM, and 24-bit PCM (scipy left-justifies it into int32)
        x = (data.astype(np.float64) / 2.0 ** 31).astype(np.float32)
    elif data.dtype in (np.float32, np.float64):
        x = data.astype(np.float32)
    else:
        raise ValueError(f"audio: unsupported WAV sample type {data.dtype} in {path!r}")
    return x, int(sr)


def resample(x, sr, target):
    """Polyphase resampling of float32 [n] from sr to target Hz; length ceil(n * target / sr) (librosa's rule)."""
    if sr == target:
        return x
    from scipy.signal import resample_poly
    g = math.gcd(int(sr), int(target))
    n_out = int(math.ceil(len(x) * target / sr))
    y = resample_poly(x.astype(np.float64), target // g, sr // g)
    if len(y) < n_out:
        y = np.pad(y, (0, n_out - len(y)))
    return y[:n_out].astype(np.float32)


def _biquad(kind, G, Q, fc, rate):
    """RBJ cookbook biquad (b, a), normalised by a0, as pyloudnorm's IIRfilter builds its K-weighting stages."""
    A = 10 ** (G / 40.0)
    w0 = 2.0 * np.pi * (fc / rate)
    alpha = np.sin(w0) / (2.0 * Q)
    c = np.cos(w0)
    if kind == "high_shelf":
        b = [A * ((A + 1) + (A - 1) * c + 2 * np.sqrt(A) * alpha), -2 * A * ((A - 1) + (A + 1) * c),
             A * ((A + 1) + (A - 1) * c - 2 * np.sqrt(A) * alpha)]
        a = [(A + 1) - (A - 1) * c + 2 * np.sqrt(A) * alpha, 2 * ((A - 1) - (A + 1) * c),
             (A + 1) - (A - 1) * c - 2 * np.sqrt(A) * alpha]
    elif kind == "high_pass":
        b = [(1 + c) / 2, -(1 + c), (1 + c) / 2]
        a = [1 + alpha, -2 * c, 1 - alpha]
    else:
        raise ValueError(kind)
    return np.array(b) / a[0], np.array(a) / a[0]


def integrated_loudness(data, rate, block_size=0.400):
    """BS.1770-4 integrated loudness (LUFS) of float samples [n] or [n, channels] (pyloudnorm Meter.integrated_loudness)."""
    from scipy.signal import lfilter
    x = np.asarray(data, dtype=np.float64)
    x = x.reshape(len(x), -1)
    for kind, G, Q, fc in (("high_shelf", 4.0, 1 / np.sqrt(2), 1500.0), ("high_pass", 0.0, 0.5, 38.0)):
        b, a = _biquad(kind, G, Q, fc, rate)
        x = lfilter(b, a, x, axis=0)
    n_ch = x.shape[1]
    step = 0.25                                                   # 75 % overlap
    T = x.shape[0] / rate
    n_blocks = int(np.round((T - block_size) / (block_size * step))) + 1
    if n_blocks < 1:
        return float("-inf")
    z = np.zeros((n_ch, n_blocks))
    for j in range(n_blocks):
        lo, hi = int(block_size * (j * step) * rate), int(block_size * (j * step + 1) * rate)
        z[:, j] = (x[lo:hi] ** 2).sum(axis=0) / (block_size * rate)
    gains = np.array([1.0, 1.0, 1.0, 1.41, 1.41][:n_ch])
    with np.errstate(divide="ignore", invalid="ignore"):
        l = -0.691 + 10.0 * np.log10((gains[:, None] * z).sum(axis=0))
        gated = l >= -70.0
        if not gated.any():
            return float("-inf")
        rel = -0.691 + 10.0 * np.log10((gains * z[:, gated].mean(axis=1)).sum()) - 10.0
        gated = (l > rel) & (l > -70.0)
        if not gated.any():
            return float("-inf")
        return float(-0.691 + 10.0 * np.log10((gains * z[:, gated].mean(axis=1)).sum()))


def loudness_norm(audio_array, sr=16000, lufs=-23):
    """reference :10-16: scale to `lufs` integrated loudness; returned unchanged when |loudness| > 100 (e.g. silence)."""
    loudness = integrated_loudness(audio_array, sr)
    if not np.isfinite(loudness) or abs(loudness) > 100:
        return audio_array
    return audio_array * (10.0 ** ((lufs - loudness) / 20.0))


def audio_prepare_single(audio_path, sample_rate=16000):
    """reference :67-75 for WAV files: mono float32 at `sample_rate`, loudness-normalised to -23 LUFS."""
    ext = os.path.splitext(audio_path)[1].lower()
    if ext not in _WAV_EXT:
        raise ValueError(f"audio: {audio_path!r}: only WAV files are read here (mp3 / m4a / flac / video containers need "
                         f"ffmpeg); convert it first, e.g. `ffmpeg -i in{ext} -ac 1 -ar {sample_rate} out.wav`")
    x, sr = read_wav(audio_path)
    if x.ndim == 2:
        x = x.mean(axis=1).astype(np.float32)                    # librosa.to_mono: channel mean
    x = resample(x, sr, sample_rate)
    return loudness_norm(x, sample_rate)


def get_embedding(speech_array, wav2vec_feature_extractor, audio_encoder, sr=16000, device="cuda"):
    """reference :18-41: wav2vec2 hidden states 1..L of a 16 kHz waveform at 25 fps -> f32 [T, L, d] on `device`,
    T = int(len / sr * 25)."""
    seq_len = int(len(speech_array) / sr * 25)
    iv = wav2vec_feature_extractor(speech_array, sampling_rate=sr).input_values
    iv = torch.from_numpy(np.squeeze(np.asarray(iv, dtype=np.float32)).reshape(-1))
    with torch.no_grad():
        out = audio_encoder.engine(device).forward(iv, seq_len, output_hidden_states=True)
    return out.stacked[1:].transpose(0, 1).contiguous()
