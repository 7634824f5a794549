"""Log-mel front end of the TTS targets on the device (SURVEY section 8a row 15; reference
speecht5/data/text_to_speech_dataset.py:95-138, whose arithmetic is librosa's): reflect-pad n_fft/2, frames of n_fft
samples every hop, periodic-hann window, |rFFT|, Slaney mel projection, log10(max(eps, .)).

The operand views are checked on the CPU through the GEMM emulator against oracle/audio_oracle.py
(tests/test_frontend_cpu.py), the device path in tests/test_frontend_gpu.py.

Device formulation: the STFT of every utterance is ONE batched wgmma GEMM -- row t of utterance b is the n_fft
contiguous samples starting at t*hop of the padded waveform (row pitch = hop: overlapping windows, no framing copy),
times a constant [2*(n_fft/2+1), n_fft] matrix holding the windowed cosine and negative sine bases -- in split precision
(hi*hi + hi*lo + lo*hi of bf16 pairs, fp32 accumulate: measured 1e-3 worst case in the log10 domain,
tests/test_kernel_algorithms_cpu.py). Magnitude and log are elementwise torch calls; the mel projection is a second
GEMM. The reference does this with numpy in the data-loader workers."""
import math

import torch

from . import kernels as K

_CONST = {}


def _hz_to_mel(f):
    f_sp, min_log_hz, logstep = 200.0 / 3, 1000.0, math.log(6.4) / 27.0
    return torch.where(f >= min_log_hz, min_log_hz / f_sp + torch.log(torch.clamp(f, min=1e-30) / min_log_hz) / logstep,
                       f / f_sp)


def _mel_to_hz(m):
    f_sp, min_log_hz, logstep = 200.0 / 3, 1000.0, math.log(6.4) / 27.0
    min_log_mel = min_log_hz / f_sp
    return torch.where(m >= min_log_mel, min_log_hz * torch.exp(logstep * (m - min_log_mel)), f_sp * m)


def slaney_mel_basis(sr, n_fft, n_mels, fmin, fmax):
    """librosa.filters.mel(htk=False, norm="slaney") from its published definition, fp64 -> [n_mels, n_fft/2+1] fp32."""
    freqs = torch.linspace(0.0, sr / 2.0, 1 + n_fft // 2, dtype=torch.float64)
    lo, hi = _hz_to_mel(torch.tensor(float(fmin), dtype=torch.float64)), _hz_to_mel(
        torch.tensor(float(fmax), dtype=torch.float64))
    mel_f = _mel_to_hz(torch.linspace(float(lo), float(hi), n_mels + 2, dtype=torch.float64))
    fdiff = mel_f[1:] - mel_f[:-1]
    ramps = mel_f[:, None] - freqs[None, :]
    lower = -ramps[:-2] / fdiff[:-1, None]
    upper = ramps[2:] / fdiff[1:, None]
    w = torch.clamp(torch.minimum(lower, upper), min=0.0)
    w = w * (2.0 / (mel_f[2:] - mel_f[:-2]))[:, None]
    return w.float()


def _pair(w2d, device):
    """(hi, lo) bf16 split of a constant fp32 matrix, rows padded to a multiple of 8 elements."""
    rows, cols = w2d.shape
    ld = (cols + 7) // 8 * 8
    src = torch.zeros((rows, ld), dtype=torch.float32, device=device)
    src[:, :cols] = w2d.to(device)
    hi = torch.empty((rows, ld), dtype=torch.bfloat16, device=device)
    lo = torch.empty_like(hi)
    K.cast_bf16(src, hi, lo)
    return hi, lo, ld


def _constants(device, sr, n_fft, n_mels, fmin, fmax):
    key = (str(device), sr, n_fft, n_mels, fmin, fmax)
    if key not in _CONST:
        nb = n_fft // 2 + 1
        n = torch.arange(n_fft, dtype=torch.float64)
        ang = 2.0 * math.pi * ((n[None, :] * torch.arange(nb, dtype=torch.float64)[:, None]) % n_fft) / n_fft
        win = 0.5 - 0.5 * torch.cos(2.0 * math.pi * n / n_fft)  # periodic hann
        dft = torch.cat([torch.cos(ang), -torch.sin(ang)], dim=0) * win[None, :]  # [2*nb, n_fft]: K-major B operand
        _CONST[key] = (_pair(dft.float(), device), _pair(slaney_mel_basis(sr, n_fft, n_mels, fmin, fmax), device))
    return _CONST[key]


def _gemm3(a_hi, a_lo, b_hi, b_lo, out, **kw):
    K.gemm(a_hi, b_hi, out, **kw)
    K.gemm(a_hi, b_lo, out, accumulate=True, **kw)
    K.gemm(a_lo, b_hi, out, accumulate=True, **kw)


def logmelfilterbank(audio, sampling_rate=16000, fft_size=1024, hop_size=256, num_mels=80, fmin=80, fmax=7600,
                     eps=1e-10):
    """audio [B, n] (or [n]) fp32 CUDA tensor of equal-length (padded) utterances -> [B, 1 + n // hop, num_mels] fp32.
    Same arguments and defaults as the reference function (text_to_speech_dataset.py:95-106)."""
    K._require_cuda(audio)
    squeeze = audio.dim() == 1
    x = (audio[None] if squeeze else audio).float()
    B, n = x.shape
    pad = fft_size // 2
    xp = torch.nn.functional.pad(x[:, None], (pad, pad), mode="reflect")[:, 0]  # [B, n + n_fft]
    L = (xp.shape[1] + 7) // 8 * 8
    buf = torch.zeros((B, L), dtype=torch.float32, device=x.device)
    buf[:, : xp.shape[1]] = xp
    hi = torch.empty((B, L), dtype=torch.bfloat16, device=x.device)
    lo = torch.empty_like(hi)
    K.cast_bf16(buf, hi, lo)
    T = 1 + n // hop_size
    nb = fft_size // 2 + 1
    (d_hi, d_lo, d_ld), (m_hi, m_lo, m_ld) = _constants(x.device, sampling_rate, fft_size, num_mels, fmin, fmax)
    ldc = (2 * nb + 7) // 8 * 8
    spec = torch.empty((B, T, ldc), dtype=torch.float32, device=x.device)
    _gemm3(hi, lo, d_hi, d_lo, spec, M=T, N=2 * nb, K=fft_size, a_ld=hop_size, b_ld=d_ld, c_ld=ldc, nb1=B, nb2=1,
           a_bs=(L, 0), b_bs=(0, 0), c_bs=(T * ldc, 0))
    mag = torch.zeros((B * T, m_ld), dtype=torch.float32, device=x.device)
    mag[:, :nb] = torch.sqrt(spec[..., :nb] ** 2 + spec[..., nb:2 * nb] ** 2).view(B * T, nb)
    g_hi = torch.empty((B * T, m_ld), dtype=torch.bfloat16, device=x.device)
    g_lo = torch.empty_like(g_hi)
    K.cast_bf16(mag, g_hi, g_lo)
    mel = torch.empty((B * T, num_mels), dtype=torch.float32, device=x.device)
    _gemm3(g_hi, g_lo, m_hi, m_lo, mel, M=B * T, N=num_mels, K=nb, a_ld=m_ld, b_ld=m_ld, c_ld=num_mels)
    out = torch.log10(torch.clamp(mel, min=eps)).view(B, T, num_mels)
    return out[0] if squeeze else out
