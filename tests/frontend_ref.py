"""fp64 statement of layer 0 of the waveform feature extractor in include/speecht5_b200.h -- st5_conv0_gn_gelu_fwd / _bwd
(Conv1d + GroupNorm with one group per channel + GELU) and st5_conv0_ln_gelu_fwd / _bwd (Conv1d + LayerNorm over the
channels of each frame + GELU) -- and elementwise error bounds for the kernels in csrc/conv_frontend.cu. CPU only (the
functions run on whatever device their inputs live on); no import of speecht5_b200.

  x[b, t, k] = wave[b, t S + k]                     (the K samples of frame t; samples past (T0 - 1) S + K unused)
  v[b, t, c] = sum_k w[c, k] x[b, t, k]
  GroupNorm  : mean / var over t per (b, c); LayerNorm: over c per (b, t). Biased variance, eps inside the sqrt.
  xhat = (v - mean) rstd;  z = xhat gamma + beta;  y = act(z)
  backward (from the SAVED mean / rstd): g = dy act'(z); dbeta += sum g; dgamma += sum g xhat;
             dv = rstd gamma (g - mean(g) - xhat mean(g xhat))  (means over the normalised axis);
             dw[c, k] += sum_{b, t} dv[b, t, c] x[b, t, k]

Bounds follow the kernels' arithmetic, in the style of tests/rowops_ref.py: each fp32 reduction is bounded by a depth
times 2^-24 times the sum of its absolute terms (not of its result: the statistics cancel), with the depth read off the
summation tree:
  GroupNorm statistics: one fp32 pass per 128-frame chunk, centred on the chunk's first frame (the pilot):
    sh = sum (v - pilot), qh = sum (v - pilot)^2, M2 = qh - sh^2 / n  -> depth C_CHUNK over sum |v - pilot|, (v - pilot)^2
    (M2 cancels when the pilot sits far from the chunk mean: the bound grows with sum (v - pilot)^2, not with M2);
    then Chan's merge of the chunks in fp64 (exact next to fp32), rounded once to fp32.
  GroupNorm backward: per-chunk fp32 sums of g and g xhat (C_CHUNK), fp64 totals, fp32 atomics over B into dgamma /
    dbeta; dw through per-chunk fp32 partials, then conv0_reduce_w_kernel: a sequential slice of ceil(rows / 32) rows
    plus 32 atomics.
  LayerNorm: a warp per frame, <= 16 values per lane then 5 shuffle levels (C_WARP); the backward's per-pair rows are
    accumulated over the frames a pair of warps visits, then summed by conv0_reduce_w_kernel (`ln_col_depth`)."""
import math

import torch

import rowops_ref as R

F64 = torch.float64
U32 = R.U32
TINY = R.TINY
C_EW = R.C_EW
TCH = 128              # frames per chunk (C0_TCH)
C_CHUNK = TCH + 4      # a chunk's sequential fp32 sums
C_WARP = 32            # one warp over <= 512 channels: 16 per lane + 5 shuffle levels (+ slack)
A2 = 1.0               # |act''| <= 0.80 for the erf GELU, <= 0.84 for the tanh form: carries an error of z into act'(z)
check = R.check
exceeds = R.exceeds


def frames(n, K, S):
    return (n - K) // S + 1 if n >= K else 0


def taps(wave, K, S):
    """x[b, t, k] = wave[b, t S + k], fp64 [B, T0, K]."""
    wave = wave.to(F64)
    T0 = frames(wave.shape[1], K, S)
    return wave[:, :(T0 - 1) * S + K].unfold(1, K, S)


def _conv(wave, w, S):
    w = w.to(F64)
    x = taps(wave, w.shape[1], S)
    return x, x @ w.T, x.abs() @ w.abs().T


def _chunks(t, T0):
    """[B, T0, C] -> [B, chunks, TCH, C] zero-padded, and the frame counts [chunks]."""
    nch = -(-T0 // TCH)
    pad = torch.zeros(t.shape[0], nch * TCH - T0, t.shape[2], dtype=t.dtype, device=t.device)
    n = torch.full((nch,), float(TCH), dtype=F64, device=t.device)
    n[-1] = T0 - (nch - 1) * TCH
    return torch.cat([t, pad], 1).view(t.shape[0], nch, TCH, t.shape[2]), n


# ============================================================================================ GroupNorm mode
def gn_forward(wave, w, gamma, beta, *, S, eps, act):
    x, v, vmag = _conv(wave, w, S)
    mean = v.mean(1)
    d = v - mean[:, None]
    var = (d * d).mean(1)
    rstd = 1.0 / torch.sqrt(var + eps)
    xhat = d * rstd[:, None]
    z = xhat * gamma.to(F64) + beta.to(F64)
    return dict(x=x, v=v, vmag=vmag, mean=mean, d=d, var=var, rstd=rstd, xhat=xhat, z=z, y=R.act(z, act),
                gamma=gamma.to(F64), beta=beta.to(F64), eps=eps, act=act, K=w.shape[1])


def _z_bound(f, ed, rstd, erstd):
    """Error of z = fma((v - mean) rstd, gamma, beta) when v - mean carries ed and rstd carries erstd."""
    g = f["gamma"].abs()
    return g * (rstd * ed + f["d"].abs() * erstd) + C_EW * U32 * ((f["xhat"] * f["gamma"]).abs() + f["z"].abs())


def gn_forward_bounds(f, u):
    """Bounds of mean, rstd [B, C] and y [B, T0, C] (storage unit u)."""
    v, T0 = f["v"], f["v"].shape[1]
    ev = f["K"] * U32 * f["vmag"]                      # the K-tap fma chain, recomputed in every pass
    vc, n = _chunks(v, T0)
    evc, _ = _chunks(ev, T0)
    live = _chunks(torch.ones_like(v[..., :1]), T0)[0]
    p, ep = vc[:, :, :1], evc[:, :, :1]
    dc = (vc - p) * live
    e_d = (evc + ep) * live
    nn_ = n[None, :, None]
    sh = dc.sum(2)
    esh = e_d.sum(2) + C_CHUNK * U32 * dc.abs().sum(2)
    es = esh + nn_ * ep[:, :, 0] + 2 * U32 * (nn_ * p[:, :, 0]).abs()                    # chunk sum fma(n, pilot, sh)
    eq = ((C_CHUNK + 4) * U32 * (dc * dc).sum(2) + 2 * (dc.abs() * e_d).sum(2)
          + (2 * sh.abs() * esh + esh * esh) / nn_)
    mu_i = vc.sum(2) / nn_
    emu = es.sum(1) / T0 + U32 * f["mean"].abs()
    evar = (eq.sum(1) + 2 * ((mu_i - f["mean"][:, None]).abs() * es).sum(1) + (es * es / nn_).sum(1)) / T0
    rstd = f["rstd"]
    erstd = rstd * (evar / (f["var"] + f["eps"]) + 2 * U32)
    ed = ev + emu[:, None] + U32 * f["d"].abs()
    ez = _z_bound(f, ed, rstd[:, None], erstd[:, None])
    ey = R.act_grad(f["z"], f["act"]).abs() * ez + A2 * ez * ez + R.act_fwd_bound(f["z"], f["act"], u)
    return dict(mean=emu + TINY, rstd=erstd + TINY, y=ey)


def _bwd_common(x, v, vmag, K, dy, gamma, beta, mean, rstd, act, axis):
    """xhat from the saved statistics, g = dy act'(z), and their error terms; axis: the normalised axis of v."""
    gamma, beta = gamma.to(F64), beta.to(F64)
    mean, rstd = mean.to(F64).unsqueeze(axis), rstd.to(F64).unsqueeze(axis)
    dy = dy.to(F64)
    d = v - mean
    xhat = d * rstd
    z = xhat * gamma + beta
    g, eg_act = R.act_bwd_bound(dy, z, act, 0.0)
    ev = K * U32 * vmag
    exh = rstd * (ev + U32 * d.abs()) + 2 * U32 * xhat.abs()
    ez = gamma.abs() * exh + 2 * U32 * ((xhat * gamma).abs() + z.abs())
    eg = eg_act + dy.abs() * A2 * ez
    return dict(x=x, dy=dy, xhat=xhat, z=z, g=g, exh=exh, eg=eg, gamma=gamma, rstd=rstd)


def gn_backward(dy, wave, w, gamma, beta, mean, rstd, *, S, act):
    """What st5_conv0_gn_gelu_bwd adds to dw, dgamma, dbeta (fp64), with the intermediates its bounds need."""
    x, v, vmag = _conv(wave, w, S)
    T0 = v.shape[1]
    b = _bwd_common(x, v, vmag, w.shape[1], dy, gamma, beta, mean, rstd, act, 1)
    g, xhat = b["g"], b["xhat"]
    S1, S2 = g.sum(1), (g * xhat).sum(1)
    m1, m2 = S1[:, None] / T0, S2[:, None] / T0
    dv = b["rstd"] * b["gamma"] * (g - m1 - xhat * m2)
    b.update(S1=S1, S2=S2, m1=m1, m2=m2, dv=dv, T0=T0, dbeta=S1.sum(0), dgamma=S2.sum(0),
             dw=torch.einsum("btc,btk->ck", dv, x))
    return b


def gn_backward_bounds(b, dw0, dgamma0, dbeta0):
    """Bounds of dw, dgamma, dbeta after the kernel adds into accumulators that held dw0, dgamma0, dbeta0."""
    g, xhat, eg, exh, T0 = b["g"], b["xhat"], b["eg"], b["exh"], b["T0"]
    B = g.shape[0]
    eS1 = C_CHUNK * U32 * g.abs().sum(1) + eg.sum(1) + U32 * b["S1"].abs()
    eS2 = C_CHUNK * U32 * (g * xhat).abs().sum(1) + (g.abs() * exh + xhat.abs() * eg).sum(1) + U32 * b["S2"].abs()
    dep = (B + 1) * U32
    edbeta = eS1.sum(0) + dep * (b["S1"].abs().sum(0) + dbeta0.abs())
    edgamma = eS2.sum(0) + dep * (b["S2"].abs().sum(0) + dgamma0.abs())
    em1 = eS1[:, None] / T0 + 2 * U32 * b["m1"].abs()
    em2 = eS2[:, None] / T0 + 2 * U32 * b["m2"].abs()
    rg = b["rstd"] * b["gamma"].abs()
    edv = rg * (eg + em1 + exh * b["m2"].abs() + xhat.abs() * em2) \
        + C_EW * U32 * rg * (g.abs() + b["m1"].abs() + (xhat * b["m2"]).abs())
    ax = b["x"].abs()
    rows = B * -(-T0 // TCH)
    depth = C_CHUNK + -(-rows // 32) + 33
    edw = depth * U32 * (torch.einsum("btc,btk->ck", b["dv"].abs(), ax) + dw0.abs()) \
        + torch.einsum("btc,btk->ck", edv, ax)
    return dict(dw=edw + TINY, dgamma=edgamma + TINY, dbeta=edbeta + TINY)


# ============================================================================================ LayerNorm mode
def ln_forward(wave, w, gamma, beta, *, S, eps, act):
    """mean / rstd flattened to [B * T0] as the kernel saves them."""
    x, v, vmag = _conv(wave, w, S)
    mean = v.mean(2)
    d = v - mean[..., None]
    var = (d * d).mean(2)
    rstd = 1.0 / torch.sqrt(var + eps)
    xhat = d * rstd[..., None]
    z = xhat * gamma.to(F64) + beta.to(F64)
    return dict(x=x, v=v, vmag=vmag, mean=mean, d=d, var=var, rstd=rstd, xhat=xhat, z=z, y=R.act(z, act),
                gamma=gamma.to(F64), beta=beta.to(F64), eps=eps, act=act, K=w.shape[1])


def ln_forward_bounds(f, u):
    C = f["v"].shape[2]
    ev = f["K"] * U32 * f["vmag"]
    d = f["d"]
    emu = (ev.sum(2) + C_WARP * U32 * f["v"].abs().sum(2)) / C + 2 * U32 * f["mean"].abs()
    ed = ev + emu[..., None] + U32 * d.abs()
    evar = (2 * (d.abs() * ed).sum(2) + (ed * ed).sum(2) + C_WARP * U32 * (d * d).sum(2)) / C + 2 * U32 * f["var"]
    rstd = f["rstd"]
    erstd = rstd * (evar / (f["var"] + f["eps"]) + 4 * U32)       # (rsqrtf: 2 ulp)
    ez = _z_bound(f, ed, rstd[..., None], erstd[..., None])
    ey = R.act_grad(f["z"], f["act"]).abs() * ez + A2 * ez * ez + R.act_fwd_bound(f["z"], f["act"], u)
    return dict(mean=emu.reshape(-1) + TINY, rstd=erstd.reshape(-1) + TINY, y=ey)


def ln_col_depth(n_frames, sms):
    """Depth of a column sum of the LayerNorm backward: the frames one pair of warps visits (persistent grid of
    min(ceil(frames / 4), 2 sms) CTAs x 4 pairs), then conv0_reduce_w_kernel over the pair rows."""
    grid = max(1, min(-(-n_frames // 4), 2 * sms))
    rows = grid * 4
    return -(-n_frames // rows) + -(-rows // 32) + 33


def ln_backward(dy, wave, w, gamma, beta, mean, rstd, *, S, act):
    """mean / rstd [B * T0] (saved); returns what st5_conv0_ln_gelu_bwd adds to dw, dgamma, dbeta (fp64)."""
    x, v, vmag = _conv(wave, w, S)
    B, T0, C = v.shape
    b = _bwd_common(x, v, vmag, w.shape[1], dy, gamma, beta, mean.reshape(B, T0), rstd.reshape(B, T0), act, 2)
    g, xhat = b["g"], b["xhat"]
    dxh = g * b["gamma"]
    m1 = dxh.mean(2, keepdim=True)
    m2 = (dxh * xhat).mean(2, keepdim=True)
    du = b["rstd"] * (dxh - m1 - xhat * m2)
    b.update(dxh=dxh, m1=m1, m2=m2, du=du, dgamma=(g * xhat).sum((0, 1)), dbeta=g.sum((0, 1)),
             dw=torch.einsum("btc,btk->ck", du, x))
    return b


def ln_backward_bounds(b, dw0, dgamma0, dbeta0, sms):
    g, xhat, eg, exh, dxh = b["g"], b["xhat"], b["eg"], b["exh"], b["dxh"]
    B, T0, C = g.shape
    edxh = b["gamma"].abs() * eg + U32 * dxh.abs()
    em1 = (edxh.sum(2, keepdim=True) + C_WARP * U32 * dxh.abs().sum(2, keepdim=True)) / C + 2 * U32 * b["m1"].abs()
    em2 = ((dxh.abs() * exh + xhat.abs() * edxh).sum(2, keepdim=True)
           + C_WARP * U32 * (dxh * xhat).abs().sum(2, keepdim=True)) / C + 2 * U32 * b["m2"].abs()
    rstd = b["rstd"]
    edu = rstd * (edxh + em1 + exh * b["m2"].abs() + xhat.abs() * em2) \
        + C_EW * U32 * rstd * (dxh.abs() + b["m1"].abs() + (xhat * b["m2"]).abs())
    dep = ln_col_depth(B * T0, sms) * U32
    ax = b["x"].abs()
    edw = dep * (torch.einsum("btc,btk->ck", b["du"].abs(), ax) + dw0.abs()) + torch.einsum("btc,btk->ck", edu, ax)
    edg = dep * ((g * xhat).abs().sum((0, 1)) + dgamma0.abs()) + (eg * xhat.abs() + g.abs() * exh).sum((0, 1))
    edb = dep * (g.abs().sum((0, 1)) + dbeta0.abs()) + eg.sum((0, 1))
    return dict(dw=edw + TINY, dgamma=edg + TINY, dbeta=edb + TINY)
