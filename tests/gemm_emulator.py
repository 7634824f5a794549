"""CPU emulation of the C-ABI entry points the host-side compositions call (st5_gemm_bf16 semantics as documented in
include/speecht5_b200.h, st5_cast_bf16, st5_act_bwd), so that the INDEX ALGEBRA of a composition -- operand views, row
pitches, batch strides, phase offsets -- can be checked on the CPU against torch. Test infrastructure only: the product
path has no CPU fallback; tests install these with monkeypatch."""
import math

import torch


def _view(t, nb1, rows, K, mn, ld, bs1, nb2=1, bs2=0):
    """[nb2 * nb1, rows, K] view of an operand (batch index z = b2 * nb1 + b1; a stride of 0 broadcasts)."""
    base = t.storage_offset()
    if mn:  # memory [K][ld], row index contiguous
        v = torch.as_strided(t, (nb2, nb1, K, rows), (bs2, bs1, ld, 1), base).transpose(2, 3)
    else:
        v = torch.as_strided(t, (nb2, nb1, rows, K), (bs2, bs1, ld, 1), base)
    return v.reshape(nb2 * nb1, rows, K)


def _gelu_grad(z):
    return 0.5 * (1 + torch.erf(z / math.sqrt(2))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)


def _tanh_u(z):
    return torch.tanh(math.sqrt(2 / math.pi) * (z + 0.044715 * z ** 3))


def _gelu_tanh(z):
    """The tanh form of GELU the kernels evaluate for act = gelu_tanh (include/speecht5_b200.h ST5_ACT_GELU_TANH)."""
    return 0.5 * z * (1 + _tanh_u(z))


def _gelu_tanh_grad(z):
    t = _tanh_u(z)
    return 0.5 * (1 + t) + 0.5 * z * (1 - t * t) * math.sqrt(2 / math.pi) * (1 + 3 * 0.044715 * z * z)


def _act(v, act):
    if act == "gelu":
        return torch.nn.functional.gelu(v)
    if act in ("gelu_tanh", "gelu_tanh_gate"):
        return _gelu_tanh(v)
    if act == "relu":
        return torch.relu(v)
    if act == "tanh":
        return torch.tanh(v)
    assert act in (None, "none"), act
    return v


def _act_grad(z, act):
    if act == "gelu":
        return _gelu_grad(z)
    if act == "gelu_tanh":
        return _gelu_tanh_grad(z)
    if act == "relu":
        return (z > 0).to(z.dtype)
    if act == "tanh":
        return 1.0 - torch.tanh(z) ** 2
    raise AssertionError(act)


def gemm_keep(M, N, nb, drop_p, seed, offset, rows=None, cols=None):
    """[nb, M, N] keep mask of the GEMM epilogue's dropout: element (z, m, n) has index (z * M + m) * N + n -- the logical
    output, whatever c_ld and the batch strides are (tests/dropout_ref.py states the generator). rows / cols (index
    tensors): the [nb, len(rows), len(cols)] part of it only."""
    import numpy as np
    import dropout_ref
    r = np.arange(M, dtype=np.uint64) if rows is None else rows.numpy().astype(np.uint64)
    c = np.arange(N, dtype=np.uint64) if cols is None else cols.numpy().astype(np.uint64)
    idx = (np.arange(nb, dtype=np.uint64)[:, None, None] * np.uint64(M) + r[:, None]) * np.uint64(N) + c
    return torch.from_numpy(dropout_ref.keep_mask(seed, offset, idx, drop_p))


def gemm(a, b, out, *, M, N, K, a_mn=False, b_mn=False, a_ld=None, b_ld=None, c_ld=None, nb1=1, nb2=1, a_bs=(0, 0),
         b_bs=(0, 0), c_bs=(0, 0), bias=None, bias2=None, bias2_rows=0, residual=None, c_pre=None, act=None, alpha=1.0,
         accumulate=False, drop_p=0.0, seed=0, offset=0, actgrad_pre=None, actgrad_act=None, rows=None, cols=None):
    """st5_gemm_bf16 in fp64: out[z] = dropout(act(alpha * A[z] B[z]^T + c_old + bias + bias2)) * act'(actgrad_pre)
    + residual, z = b2 * nb1 + b1; c_pre receives the value before act() (for gelu_tanh_gate: keep * scale *
    gelu_tanh'(x) instead). bias2 row m is bias2[m // bias2_rows] at a row pitch of N, the same for every batch entry
    (the kernel does not index it by z). rows / cols (index tensors into [M) / [N)): compute and write only the outputs
    (z, rows[i], cols[j]) -- every output depends on its own row of A and column of B^T only, over the full K."""
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16
    assert not (int(offset) >> 63), "device-resident seeds: pass the seed value itself"
    a_ld = a_ld if a_ld is not None else (M if a_mn else K)
    b_ld = b_ld if b_ld is not None else (N if b_mn else K)
    c_ld = c_ld if c_ld is not None else N
    for t, ld, bs in ((a, a_ld, a_bs), (b, b_ld, b_bs)):  # what cuTensorMapEncodeTiled demands of an operand
        assert (t.storage_offset() * 2) % 16 == 0 and (ld * 2) % 16 == 0, "TMA alignment"
        assert (bs[0] * 2) % 16 == 0 and (bs[1] * 2) % 16 == 0, "TMA alignment"
    nb = nb1 * nb2
    rr = torch.arange(M) if rows is None else rows
    cc = torch.arange(N) if cols is None else cols
    A = _view(a, nb1, M, K, a_mn, a_ld, a_bs[0], nb2, a_bs[1])[:, rr].double()
    B = _view(b, nb1, N, K, b_mn, b_ld, b_bs[0], nb2, b_bs[1])[:, cc].double()
    Mr, Nc = len(rr), len(cc)
    v = (alpha * torch.bmm(A, B.transpose(1, 2))).reshape(nb2, nb1, Mr, Nc)
    sub = (slice(None), slice(None), rr[:, None], cc[None, :])

    def out_view(t):
        return torch.as_strided(t, (nb2, nb1, M, N), (c_bs[1], c_bs[0], c_ld, 1), t.storage_offset())

    def read(t):
        return out_view(t)[sub]

    def write(t, val):
        out_view(t)[sub] = val.to(t.dtype)
    shared = (nb1 > 1 and c_bs[0] == 0) or (nb2 > 1 and c_bs[1] == 0)
    if int(accumulate) == 2:  # L2-side accumulate: batch entries may share one output (c_bs = 0), split-K
        assert out.dtype == torch.float32 and (c_ld * 4) % 16 == 0 and bias is None and c_pre is None and act in (None, "none")
        assert bias2 is None and residual is None and actgrad_pre is None and drop_p == 0.0
        C = out_view(out)
        for b2 in range(nb2):
            for b1 in range(nb1):
                C[b2, b1][sub[2:]] = (C[b2, b1][sub[2:]].double() + v[b2, b1]).to(out.dtype)
        return out
    assert not shared, "several batch entries into one output need accumulate = 2"
    assert not (accumulate and out.dtype == torch.bfloat16), "accumulate needs an fp32 output"
    if accumulate:
        v = v + read(out).double()
    if bias is not None:
        assert bias.dtype == torch.float32
        v = v + bias[:N][cc].double()
    if bias2 is not None:  # per-utterance bias: row m takes bias2[m // bias2_rows], row pitch N
        assert bias2.dtype == torch.float32 and bias2_rows > 0
        flat = bias2.reshape(-1).double()
        v = v + flat[(rr // bias2_rows)[:, None] * N + cc]
    keep = gemm_keep(M, N, nb, drop_p, seed, offset, rows, cols).reshape(nb2, nb1, Mr, Nc) if drop_p > 0 else None
    scale = 1.0 / (1.0 - drop_p) if drop_p > 0 else 1.0
    if act == "gelu_tanh_gate":
        assert c_pre is not None and out.dtype == torch.bfloat16 and N % 8 == 0
        second = _gelu_tanh_grad(v) * (keep * scale if keep is not None else 1.0)  # the backward multiplier
        write(c_pre, second)
    elif c_pre is not None:
        write(c_pre, v)
    v = _act(v, act)
    if keep is not None:
        v = torch.where(keep, v * scale, torch.zeros_like(v))
    if actgrad_pre is not None:  # activation backward fused into the product: v *= act'(pre[m][n])
        pre = read(actgrad_pre).double()
        v = v * (pre if actgrad_act == "gate" else _act_grad(pre, actgrad_act))
    if residual is not None:  # same layout and dtype as C, added after the activation
        assert residual.dtype == out.dtype
        v = v + read(residual).double()
    write(out, v)
    return out


def cast_bf16(src, hi, lo=None):
    h = src.to(torch.bfloat16)
    hi.copy_(h)
    if lo is not None:
        lo.copy_((src - h.float()).to(torch.bfloat16))


def lrelu_pad(x, out, d, ph, pad, slope):
    """st5_lrelu_pad: out[b, m] = leaky_relu(x[b, ph + d*m - pad]) inside [0, T), zeros outside."""
    B, T, C = x.shape
    n_in = out.shape[1]
    idx = ph + d * torch.arange(n_in) - pad
    ok = (idx >= 0) & (idx < T)
    out.zero_()
    v = x[:, idx[ok]].float()
    out[:, ok] = torch.where(v > 0, v, v * slope).to(out.dtype)


def act_bwd(dy, pre, dpre, act, drop_p=0.0, seed=0, offset=0):
    """st5_act_bwd: dpre = dropout-backward(dy) * act'(pre), dropout index = linear element index."""
    g = dy.double()
    if drop_p > 0:
        import numpy as np
        import dropout_ref
        keep = torch.from_numpy(dropout_ref.keep_mask(seed, offset, np.arange(dy.numel(), dtype=np.uint64), drop_p))
        g = torch.where(keep.reshape(dy.shape), g / (1.0 - drop_p), torch.zeros_like(g))
    dpre.copy_((g * _act_grad(pre.double(), act)).to(dpre.dtype))


def colsum(x2d, out, group_rows=0, accumulate=False, ld=None):
    """st5_colsum: out[g][n] (+)= sum of the rows of group g (groups of `group_rows` consecutive rows; 0 = one group)."""
    rows, cols = x2d.shape
    assert ld is None or rows <= 1 or ld == x2d.stride(0)
    xs = x2d.double()
    if group_rows and group_rows > 0:
        ng = (rows + group_rows - 1) // group_rows
        padded = torch.zeros((ng * group_rows, cols), dtype=torch.float64)
        padded[:rows] = xs
        tot = padded.view(ng, group_rows, cols).sum(1)
    else:
        tot = xs.sum(0)
    flat = out.reshape(-1)
    flat.copy_(((flat.double() if accumulate else 0) + tot.reshape(-1)).to(out.dtype))


def ln_fwd(x, residual, gamma, beta, y, s_out, mean, rstd, eps, drop_p=0.0, seed=0, offset=0, residual_f32=None,
           y_f32=None):
    """st5_ln_fwd / st5_ln_fwd_stream without dropout: s = x (+ residual), y = LayerNorm(s) over the last dimension."""
    assert drop_p == 0.0
    res = residual_f32 if residual_f32 is not None else residual
    s_ = x.double() + (res.double() if res is not None else 0.0)
    mu = s_.mean(-1, keepdim=True)
    var = s_.var(-1, unbiased=False, keepdim=True)
    rs = 1.0 / torch.sqrt(var + eps)
    y.copy_(((s_ - mu) * rs * gamma.double() + beta.double()).to(y.dtype))
    if y_f32 is not None:
        y_f32.copy_(((s_ - mu) * rs * gamma.double() + beta.double()).float())
    if s_out is not None:
        s_out.copy_(s_.to(s_out.dtype))
    mean.copy_(mu.reshape(-1).float())
    rstd.copy_(rs.reshape(-1).float())


def ln_bwd(dy, s, mean, rstd, gamma, ds, dx, dgamma, dbeta, drop_p=0.0, seed=0, offset=0, dxsum=None):
    """st5_ln_bwd without dropout: ds (= dx), dgamma / dbeta accumulated, dxsum += column sums of dx (the producing
    projection's bias gradient, include/speecht5_b200.h)."""
    assert drop_p == 0.0
    C = dy.shape[-1]
    d = dy.double().reshape(-1, C)
    xh = (s.double().reshape(-1, C) - mean.double()[:, None]) * rstd.double()[:, None]
    g = d * gamma.double()
    r = rstd.double()[:, None] * (g - g.mean(-1, keepdim=True) - xh * (g * xh).mean(-1, keepdim=True))
    if ds is not None:
        ds.copy_(r.reshape(ds.shape).to(ds.dtype))
    if dx is not None:
        dx.copy_(r.reshape(dx.shape).to(dx.dtype))
    if dgamma is not None:
        dgamma.add_((d * xh).sum(0).float())
    if dbeta is not None:
        dbeta.add_(d.sum(0).float())
    if dxsum is not None:
        dxsum[:C].add_(r.sum(0).float())


def conv0_gn_gelu_fwd(wave, w, gamma, beta, y, mean, rstd, stride, eps, act):
    """st5_conv0_gn_gelu_fwd: Conv1d(1 -> C, k, stride) + GroupNorm(C groups) + GELU, channels-last output."""
    v = torch.nn.functional.conv1d(wave.double()[:, None], w.double()[:, None], stride=stride)  # [B, C, T0]
    mu = v.mean(-1)
    var = v.var(-1, unbiased=False)
    rs = 1.0 / torch.sqrt(var + eps)
    z = (v - mu[..., None]) * rs[..., None] * gamma.double()[None, :, None] + beta.double()[None, :, None]
    y.copy_(torch.nn.functional.gelu(z).transpose(1, 2).to(y.dtype))
    mean.copy_(mu.float())
    rstd.copy_(rs.float())


def _conv0_ln(wave, w, gamma, beta, eps):
    v = torch.nn.functional.conv1d(wave.double()[:, None], w[:, None], stride=_conv0_ln.stride).transpose(1, 2)  # [B, T0, C]
    return v, torch.nn.functional.layer_norm(v, (v.shape[-1],), gamma, beta, eps)


def conv0_ln_gelu_fwd(wave, w, gamma, beta, y, mean, rstd, stride, eps, act):
    """st5_conv0_ln_gelu_fwd: Conv1d(1 -> C, k, stride) + LayerNorm over the channels of each frame + GELU."""
    _conv0_ln.stride = stride
    v, z = _conv0_ln(wave, w.double(), gamma.double(), beta.double(), eps)
    y.copy_(torch.nn.functional.gelu(z).to(y.dtype))
    mean.copy_(v.mean(-1).reshape(-1).float())
    rstd.copy_((1.0 / torch.sqrt(v.var(-1, unbiased=False) + eps)).reshape(-1).float())


def conv0_ln_gelu_bwd(dy, wave, w, gamma, beta, mean, rstd, dw, dgamma, dbeta, stride, act):
    """st5_conv0_ln_gelu_bwd via autograd on the torch statement of the layer; dw / dgamma / dbeta accumulate."""
    _conv0_ln.stride = stride
    w_, g_, b_ = (t.double().clone().requires_grad_() for t in (w, gamma, beta))
    with torch.enable_grad():
        y = torch.nn.functional.gelu(_conv0_ln(wave, w_, g_, b_, 1e-5)[1])
        gw, gg, gb = torch.autograd.grad(y, (w_, g_, b_), dy.double())
    dw.add_(gw.float())
    dgamma.add_(gg.float())
    dbeta.add_(gb.float())


def act_fwd(x, y, act):
    assert act in ("gelu", "gelu_tanh")
    y.copy_(torch.nn.functional.gelu(x.double()).to(y.dtype))


def posenc_fwd(tokens, emb, x, pe, alpha, y, drop_p=0.0, seed=0, offset=0):
    """st5_posenc_fwd without dropout: y[b, t] = (emb[tokens[b, t]] | x[b, t]) + alpha * pe[t]."""
    assert drop_p == 0.0
    T = y.shape[1]
    base = emb.double()[tokens] if tokens is not None else x.double()
    y.copy_((base + alpha.double() * pe.double()[:T][None]).to(y.dtype))


def attention(q_buf, kv_buf, *, H, d, q_col, k_col, v_col, scale, pe_k=None, maxpos=0, key_pad=None, causal=False,
              drop_p=0.0, return_probs=False):
    """ops.attention (forward, no dropout) restated with torch: multihead_attention.py:340-389 incl. the relative-position
    bias q_i . pe[clamp(i - j, -maxpos, maxpos - 1) + maxpos] (q already scaled)."""
    assert drop_p == 0.0
    kvb = q_buf if kv_buf is None else kv_buf
    B, Tq, Tk = q_buf.shape[0], q_buf.shape[1], kvb.shape[1]

    def heads(buf, col, T):
        return buf[..., col * d:(col + 1) * d].double().reshape(B, T, H, d // H).transpose(1, 2)
    q, k, v = heads(q_buf, q_col, Tq) * scale, heads(kvb, k_col, Tk), heads(kvb, v_col, Tk)
    s = q @ k.transpose(-1, -2)
    if pe_k is not None:
        i = torch.arange(Tq)[:, None]
        j = torch.arange(Tk)[None, :]
        pos = pe_k.double()[(i - j).clamp(-maxpos, maxpos - 1) + maxpos]  # [Tq, Tk, 64]
        s = s + torch.einsum("bhic,ijc->bhij", q, pos)
    if causal:
        s = s + torch.triu(torch.full((Tq, Tk), float("-inf"), dtype=s.dtype), 1)
    if key_pad is not None:
        s = s.masked_fill(key_pad.bool()[:, None, None, :], float("-inf"))
    p = torch.softmax(s, -1)
    out = (p @ v).transpose(1, 2).reshape(B, Tq, d).to(q_buf.dtype)
    return out, (p.float() if return_probs else None)


def bn_fwd(x, x_ld, gamma, beta, running_mean, running_var, save_mean, save_rstd, y, y_ld, y_pre, rows, Cc, training,
           momentum, eps, act, drop_p, seed, offset, scratch):
    """st5_bn_fwd without dropout: BatchNorm1d over all rows of a channels-last [rows, C] tensor (+ tanh)."""
    assert drop_p == 0.0 and x_ld == Cc and y_ld == Cc
    xs = x.double().reshape(rows, Cc)
    if training:
        mu, var = xs.mean(0), xs.var(0, unbiased=False)
    else:
        mu, var = running_mean.double(), running_var.double()
    rs = 1.0 / torch.sqrt(var + eps)
    pre = (xs - mu) * rs * gamma.double() + beta.double()
    if y_pre is not None:
        y_pre.copy_(pre.reshape(y_pre.shape).to(y_pre.dtype))
    out = torch.tanh(pre) if act == "tanh" else pre
    assert act in (None, "none", "tanh")
    y.copy_(out.reshape(y.shape).to(y.dtype))
    save_mean.copy_(mu.float())
    save_rstd.copy_(rs.float())


def conv0_gn_gelu_bwd(dy, wave, w, gamma, beta, mean, rstd, dw, dgamma, dbeta, stride, act):
    """st5_conv0_gn_gelu_bwd via autograd on the torch statement of the layer; dw / dgamma / dbeta accumulate."""
    w_, g_, b_ = (t.double().clone().requires_grad_() for t in (w, gamma, beta))
    with torch.enable_grad():
        v = torch.nn.functional.conv1d(wave.double()[:, None], w_[:, None], stride=stride)
        y = torch.nn.functional.gelu(torch.nn.functional.group_norm(v, w.shape[0], g_, b_, 1e-5)).transpose(1, 2)
        gw, gg, gb = torch.autograd.grad(y, (w_, g_, b_), dy.double())
    dw.add_(gw.float())
    dgamma.add_(gg.float())
    dbeta.add_(gb.float())


def residual_layer_norm(x, residual, ln, drop_p=0.0, stream=False):
    """ops.residual_layer_norm as differentiable torch ops (for CPU checks of whole training steps)."""
    assert drop_p == 0.0
    s_ = x if residual is None else x + residual
    return torch.nn.functional.layer_norm(s_.float(), (s_.shape[-1],), ln.weight, ln.bias, ln.eps).to(x.dtype)


def scaled_posenc(pe, alpha, drop_p, tokens=None, emb=None, padding_idx=None, x=None):
    """ops.scaled_posenc as differentiable torch ops."""
    assert drop_p == 0.0
    base = torch.nn.functional.embedding(tokens, emb, padding_idx) if tokens is not None else x
    T = base.shape[1]
    from speecht5_b200.ops import RT
    return (base.float() + alpha * pe[:T][None]).to(RT.dtype)


def install_autograd(monkeypatch):
    """install() plus differentiable torch stand-ins for the ops whose backward kernels are not emulated (LayerNorm,
    embedding + positions; the emulated attention is already plain torch): whole training steps can then be
    back-propagated on the CPU, with LinearFn / FFNFn / the front-end Functions still running their own backward
    compositions on the emulated GEMM."""
    install(monkeypatch)
    from speecht5_b200 import kernels as K, ops
    monkeypatch.setattr(K, "conv0_gn_gelu_bwd", conv0_gn_gelu_bwd)
    monkeypatch.setattr(K, "conv0_ln_gelu_bwd", conv0_ln_gelu_bwd)
    monkeypatch.setattr(ops, "residual_layer_norm", residual_layer_norm)
    monkeypatch.setattr(ops, "scaled_posenc", scaled_posenc)


def install(monkeypatch):
    from speecht5_b200 import kernels as K
    monkeypatch.setattr(K, "gemm", gemm)
    monkeypatch.setattr(K, "cast_bf16", cast_bf16)
    monkeypatch.setattr(K, "act_bwd", act_bwd)
    monkeypatch.setattr(K, "lrelu_pad", lrelu_pad)
    monkeypatch.setattr(K, "colsum", colsum)
    monkeypatch.setattr(K, "ln_fwd", ln_fwd)
    monkeypatch.setattr(K, "ln_bwd", ln_bwd)
    monkeypatch.setattr(K, "posenc_fwd", posenc_fwd)
    monkeypatch.setattr(K, "bn_fwd", bn_fwd)
    from speecht5_b200 import ops
    monkeypatch.setattr(ops, "attention", attention)
    monkeypatch.setattr(K, "conv0_gn_gelu_fwd", conv0_gn_gelu_fwd)
    monkeypatch.setattr(K, "conv0_ln_gelu_fwd", conv0_ln_gelu_fwd)
    monkeypatch.setattr(K, "act_fwd", act_fwd)
    monkeypatch.setattr(K, "_require_cuda", lambda *ts: None)


# ---------------------------------------------------------------------------------------------- optimizer (csrc/optim.cu)
def sumsq(x, out):
    out += (x.double() ** 2).sum().float()


def adam_step(p, g, m, v, p_bf16, lr, beta1, beta2, eps, weight_decay, step, grad_norm_sq, max_norm, grad_mul,
              lr_dev=None, step_dev=None):
    """st5_adam_step semantics: skip on a non-finite norm; clip coefficient max_norm / (norm * grad_mul + 1e-6) capped
    at 1; fairseq Adam (denominator sqrt(v) + eps, bias-corrected step size); bf16 shadow refresh."""
    import math
    if grad_norm_sq is not None and not bool(torch.isfinite(grad_norm_sq).all()):
        return
    if lr_dev is not None:
        lr = float(lr_dev)
    t = float(step_dev) if step_dev is not None else float(step)
    step_size = lr * math.sqrt(1.0 - beta2 ** t) / (1.0 - beta1 ** t)
    gscale = grad_mul
    if grad_norm_sq is not None and max_norm > 0:
        norm = float(grad_norm_sq.sqrt()) * grad_mul
        gscale *= min(1.0, max_norm / (norm + 1e-6))
    gi = g * gscale
    m.mul_(beta1).add_(gi, alpha=1 - beta1)
    v.mul_(beta2).addcmul_(gi, gi, value=1 - beta2)
    if weight_decay != 0:
        p.mul_(1 - weight_decay * lr)
    p.addcdiv_(m, v.sqrt() + eps, value=-step_size)
    if p_bf16 is not None:
        p_bf16.copy_(p.to(torch.bfloat16))


def install_trainer(monkeypatch):
    """install_autograd() + the optimizer kernels + BatchNorm as a torch call: B200Trainer runs whole updates on CPU."""
    install_autograd(monkeypatch)
    import torch.nn.functional as F
    from speecht5_b200 import kernels as K, ops
    monkeypatch.setattr(K, "sumsq", sumsq)
    monkeypatch.setattr(K, "adam_step", adam_step)

    def batch_norm_act(x, bn, training, act=None, drop_p=0.0):
        assert drop_p == 0.0 and training
        y = F.batch_norm(x.float().reshape(-1, x.shape[-1]), None, None, bn.weight, bn.bias, True, 0.0, bn.eps)
        y = torch.tanh(y) if act == "tanh" else y
        return y.reshape(x.shape).to(x.dtype)
    monkeypatch.setattr(ops, "batch_norm_act", batch_norm_act)


class Patcher:
    """monkeypatch stand-in for spawned worker processes (no pytest fixture there)."""

    def setattr(self, obj, name, value):
        setattr(obj, name, value)
