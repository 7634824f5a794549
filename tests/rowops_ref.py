"""fp64 statement of the row and elementwise entry points of include/speecht5_b200.h -- LayerNorm (st5_ln_fwd,
st5_ln_fwd_stream, st5_ln_bwd), BatchNorm (st5_bn_fwd / _bwd), st5_posenc_fwd / _bwd, st5_colsum, st5_cast_bf16,
st5_act_fwd / st5_act_bwd, st5_lrelu_pad, st5_dropout, st5_sumsq and st5_adam_step -- and elementwise error bounds for
the kernels that implement them. CPU only; no import of speecht5_b200.

Inputs are fp64 copies of exactly the values a kernel reads (bf16 operands widened, fp32 hyper-parameters as fp32).
Dropout masks come from tests/dropout_ref.py at the logical index of each element (row * C + c).

Bounds are built like tests/attention_ref.py: unit roundoff times an fp64 magnitude product of the same operands,
elementwise. Every fp32 reduction is bounded by (depth) * 2^-24 * sum |terms| -- scaled by the terms, not by the result,
because LayerNorm's mean and BatchNorm's sums cancel -- with the depth a named constant per kind of reduction:
  C_ROW  one warp over a row of <= 1024 channels (<= 32 terms per lane + a 5-level shuffle tree);
  C_COL  a column over rows: per-thread partial sums, an 8-way shared-memory step, then fp32 atomics across up to
         ~600 row blocks (BatchNorm backward at 32k rows), so the depth is the block count;
  C_GRID a whole tensor into one float: per-thread sums, block trees and one atomic per block (<= 132 * 32 blocks);
  C_EW   the few fp32 operations of an elementwise formula.
They are worst-case depths, not fitted numbers; the GPU test prints the largest err / bound it sees. On an H100 80GB
HBM3: 0.24 for the fp32 reductions (LayerNorm dgamma in bf16), 0.43 for rstd, 0.26 for Adam; the terms that only bound
one bf16 rounding (u |ref|) reach 0.99 by construction."""
import math

import numpy as np
import torch

import dropout_ref as D

F64 = torch.float64
U32 = 2.0 ** -24
U_BF16 = 2.0 ** -8
TINY = 2.0 ** -60
C_ROW = 64
C_COL = 1024
C_GRID = 8192
C_EW = 8
# A&S 7.1.26 erf (|error| <= 1.5e-7) evaluated with rcp.approx / ex2.approx (csrc/kernels.cuh gauss_cdf): error of the
# fp32 GELU Phi(x) as an absolute error of Phi; the GELU's error is |x| times it.
E_PHI = 2.5e-7
# tanh.approx.f32 (MUFU): relative error <= 2^-10.987 (PTX ISA); used by ST5_ACT_GELU_TANH and the bf16 BatchNorm tanh.
E_TANH_APPROX = 2.0 ** -10.98
# ST5_ACT_GELU_TANH against the exact erf GELU: |err| <= GELU_TANH_ABS + GELU_TANH_REL |y| (the tanh-form formula,
# 4.73e-4 at x = 2.70, plus tanh.approx's relative error on the 0.5 x tanh(.) term).
GELU_TANH_ABS = 4.8e-4
GELU_TANH_REL = 2.0 ** -10.98


def unit(dtype):
    return U_BF16 if dtype == torch.bfloat16 else U32


def f32(v):
    """A host float as the fp32 the kernel receives."""
    return float(np.float32(v))


def keep(shape, p, seed, offset):
    """Dropout keep mask of a tensor of `shape`, element index = its row-major linear index."""
    n = math.prod(shape)
    if D.drop_threshold(p) == 0:
        return torch.ones(shape, dtype=torch.bool)
    return torch.from_numpy(D.keep_mask(seed, offset, np.arange(n, dtype=np.uint64), p)).view(shape)


def check(name, got, ref, bound, report=None):
    """Assert |got - ref| <= bound elementwise (NaN / inf in got fails). Names the first failing index and the largest
    err / bound; returns that ratio (and records it in `report[name]`)."""
    got = torch.as_tensor(got).to(F64)
    ref = torch.as_tensor(ref).to(F64)
    bound = torch.as_tensor(bound).to(F64).expand_as(ref)
    err = (got - ref).abs()
    ratio = err / bound
    ratio = torch.where(torch.isfinite(got), ratio, torch.full_like(ratio, math.inf))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if report is not None:
        report[name] = max(report.get(name, 0.0), worst)
    if not worst <= 1.0:
        bad = torch.nonzero(~(ratio <= 1.0))
        first = tuple(int(t) for t in bad[0])
        raise AssertionError(f"{name}: {bad.shape[0]} of {ratio.numel()} elements out of bound; first {first}: "
                             f"got {float(got[first]):.6g} ref {float(ref[first]):.6g} bound "
                             f"{float(bound[first]):.3g}; max err/bound {worst:.3g}")
    return worst


def exceeds(got, ref, bound):
    """True when some element of got leaves the bound (for showing that a defect would be caught)."""
    try:
        check("defect", got, ref, bound)
    except AssertionError:
        return True
    return False


# ============================================================================================ LayerNorm
def ln_forward(x, gamma, beta, *, eps, residual=None, kp=None, dscale=1.0):
    """s = residual + dropout(x); y = (s - mean) * rstd * gamma + beta over the last dim, biased variance, eps inside
    the square root. x / residual [rows, C] (residual_f32 of st5_ln_fwd_stream is just an fp32 residual)."""
    x = x.to(F64)
    xd = x * kp * dscale if kp is not None else x
    s = xd + residual.to(F64) if residual is not None else xd
    mean = s.mean(-1, keepdim=True)
    d = s - mean
    var = (d * d).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    xhat = d * rstd
    y = xhat * gamma.to(F64) + beta.to(F64)
    return dict(xd=xd, s=s, mean=mean[:, 0], rstd=rstd[:, 0], d=d, var=var, xhat=xhat, y=y, gamma=gamma.to(F64),
                beta=beta.to(F64), eps=eps)


def ln_forward_bounds(f, u):
    """Bounds of s_out (storage u), mean, rstd, y_f32 (fp32, not rounded) and y (storage u)."""
    C = f["s"].shape[-1]
    s, d, xhat, g, y = f["s"], f["d"], f["xhat"], f["gamma"], f["y"]
    rstd, var = f["rstd"][:, None], f["var"]
    es = 2 * U32 * (f["xd"].abs() + s.abs())                             # dropout scale, residual add
    emu = (C_ROW * U32 * s.abs().sum(-1, keepdim=True) + es.sum(-1, keepdim=True)) / C + U32 * f["mean"][:, None].abs()
    ed = emu + es + U32 * d.abs()
    evar = (2 * (d.abs() * ed).sum(-1, keepdim=True) + (ed * ed).sum(-1, keepdim=True)
            + C_ROW * U32 * (d * d).sum(-1, keepdim=True)) / C + U32 * var
    erstd = rstd * (0.5 * evar / (var + f["eps"]) + 4 * U32)
    ey = g.abs() * (ed * rstd + d.abs() * erstd) + C_EW * U32 * ((xhat * g).abs() + y.abs()) + TINY
    return dict(s=es + u * s.abs() + TINY, mean=emu[:, 0] + TINY, rstd=erstd[:, 0] + TINY, y_f32=ey,
                y=ey + u * y.abs())


def ln_backward(dy, s, mean, rstd, gamma, *, kp=None, dscale=1.0, dx_null=False):
    """ds = rstd (g - mean(g) - xhat mean(g xhat)), g = dy gamma, xhat = (s - mean) rstd from the SAVED mean / rstd;
    dx = dropout_bwd(ds); dgamma = sum_rows dy xhat, dbeta = sum_rows dy; dxsum = column sums of dx (of ds when dx is
    NULL). The parameter sums are what st5_ln_bwd adds to its accumulators."""
    dy, s, gamma = dy.to(F64), s.to(F64), gamma.to(F64)
    mean, rstd = mean.to(F64)[:, None], rstd.to(F64)[:, None]
    xhat = (s - mean) * rstd
    g = dy * gamma
    c1 = g.mean(-1, keepdim=True)
    c2 = (g * xhat).mean(-1, keepdim=True)
    ds = rstd * (g - c1 - xhat * c2)
    dx = ds * kp * dscale if kp is not None else ds
    return dict(dy=dy, xhat=xhat, g=g, c1=c1, c2=c2, rstd=rstd, ds=ds, dx=dx, kp=kp, dscale=dscale,
                dgamma=(dy * xhat).sum(0), dbeta=dy.sum(0), dxsum=(ds if dx_null else dx).sum(0))


def ln_backward_bounds(b, u, dx_null=False):
    C = b["ds"].shape[-1]
    xhat, g, rstd, dy = b["xhat"], b["g"], b["rstd"], b["dy"]
    exh = 3 * U32 * xhat.abs()
    eg = U32 * g.abs()
    ec1 = (C_ROW * U32 * g.abs().sum(-1, keepdim=True) + eg.sum(-1, keepdim=True)) / C
    ec2 = (C_ROW * U32 * (g * xhat).abs().sum(-1, keepdim=True)
           + (g.abs() * exh + xhat.abs() * eg).sum(-1, keepdim=True)) / C
    eds = (rstd * (eg + ec1 + exh * b["c2"].abs() + xhat.abs() * ec2)
           + C_EW * U32 * rstd * (g.abs() + b["c1"].abs() + (xhat * b["c2"]).abs()))
    sc = b["kp"] * b["dscale"] if b["kp"] is not None else 1.0
    edx = eds * sc + U32 * b["dx"].abs()
    esum = eds if dx_null else edx
    val = b["ds"] if dx_null else b["dx"]
    return dict(ds=eds + u * b["ds"].abs() + TINY, dx=edx + u * b["dx"].abs() + TINY,
                dgamma=C_COL * U32 * (dy * xhat).abs().sum(0) + (dy.abs() * exh).sum(0) + TINY,
                dbeta=C_COL * U32 * dy.abs().sum(0) + TINY,
                dxsum=C_COL * U32 * val.abs().sum(0) + esum.sum(0) + TINY)


# ============================================================================================ activations
def gelu(x):
    x = x.to(F64)
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_grad(x):
    x = x.to(F64)
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def gelu_tanh(x):
    x = x.to(F64)
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))


def gelu_tanh_grad(x):
    x = x.to(F64)
    t = torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3))
    return 0.5 * (1.0 + t) + 0.5 * x * (1.0 - t * t) * math.sqrt(2.0 / math.pi) * (1.0 + 3 * 0.044715 * x * x)


def act(x, a):
    """y = act(x) in fp64, `a` one of none / relu / gelu / tanh / gelu_tanh. The reference for gelu_tanh is the erf
    GELU the kernel stands in for (its bound carries the difference)."""
    x = x.to(F64)
    if a == "relu":
        return torch.where(x > 0, x, torch.zeros_like(x))
    if a in ("gelu", "gelu_tanh"):
        return gelu(x)
    if a == "tanh":
        return torch.tanh(x)
    return x


def act_grad(x, a):
    """act'(x); relu'(0) = 0 (torch's threshold_backward); gelu_tanh: the derivative of the tanh form it computes."""
    x = x.to(F64)
    if a == "relu":
        return (x > 0).to(F64)
    if a == "gelu":
        return gelu_grad(x)
    if a == "gelu_tanh":
        return gelu_tanh_grad(x)
    if a == "tanh":
        return 1.0 - torch.tanh(x) ** 2
    return torch.ones_like(x)


def act_fwd_bound(x, a, u):
    """|kernel - act(x)| for a finite input x (storage unit u of the output)."""
    x = x.to(F64)
    y = act(x, a)
    if a == "gelu":
        e = x.abs() * E_PHI + C_EW * U32 * y.abs()
    elif a == "gelu_tanh":
        e = GELU_TANH_ABS + GELU_TANH_REL * y.abs() + C_EW * U32 * y.abs()
    elif a == "tanh":
        e = 4 * U32 * y.abs()
    else:
        e = torch.zeros_like(y)
    return e + u * y.abs() + TINY


def act_bwd_bound(g, x, a, u):
    """|kernel - g act'(x)| where g = dropout_bwd(dy) (exact up to the fp32 scale product)."""
    x, g = x.to(F64), g.to(F64)
    d = act_grad(x, a)
    if a == "gelu":
        ed = 4 * E_PHI * (1.0 + x.abs()) + C_EW * U32 * (d.abs() + 1.0)
    elif a == "gelu_tanh":  # tanh.approx in t and in 1 - t^2
        t = torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)).abs()
        ed = E_TANH_APPROX * t * (0.5 + x.abs() * t * math.sqrt(2.0 / math.pi) * (1.0 + 0.134145 * x * x)) \
            + C_EW * U32 * (d.abs() + 1.0)
    elif a == "tanh":
        ed = 8 * U32 * (torch.tanh(x) ** 2 + d.abs())
    else:
        ed = torch.zeros_like(d)
    ref = g * d
    return ref, g.abs() * ed + 2 * U32 * ref.abs() + u * ref.abs() + TINY


def lrelu_pad(x, n_in, d, ph, pad, slope):
    """out[b][m] = leaky_relu(x[b][ph + d m - pad], slope) for source frames inside [0, T), zeros elsewhere."""
    x = x.to(F64)
    B, T, C = x.shape
    out = torch.zeros(B, n_in, C, dtype=F64)
    src = ph + d * torch.arange(n_in) - pad
    ok = (src >= 0) & (src < T)
    v = x[:, src[ok]]
    out[:, ok] = torch.where(v > 0, v, v * f32(slope))
    return out


# ============================================================================================ BatchNorm
def bn_forward(x, gamma, beta, running_mean, running_var, *, training, momentum, eps, act_name="none", kp=None,
               dscale=1.0):
    """x [rows, C]. Training: batch mean and BIASED variance normalise (eps inside the sqrt); the running variance
    takes the UNBIASED one (rows = 1: the biased 0). Eval: the running statistics normalise. pre = xhat gamma + beta,
    y = dropout(act(pre)) with the dropout index row * C + c."""
    x = x.to(F64)
    rows = x.shape[0]
    rm, rv = running_mean.to(F64), running_var.to(F64)
    out = {}
    if training:
        mu = x.mean(0)
        ss = ((x - mu) ** 2).sum(0)
        var = ss / rows
        unb = ss / (rows - 1) if rows > 1 else var
        out["running_mean"] = (1 - momentum) * rm + momentum * mu
        out["running_var"] = (1 - momentum) * rv + momentum * unb
    else:
        mu, var = rm, rv
    rstd = 1.0 / torch.sqrt(var + eps)
    xhat = (x - mu) * rstd
    pre = xhat * gamma.to(F64) + beta.to(F64)
    a = act(pre, act_name)
    y = a * kp * dscale if kp is not None else a
    out.update(x=x, mean=mu, var=var, rstd=rstd, xhat=xhat, pre=pre, a=a, y=y, gamma=gamma.to(F64), eps=eps,
               training=training, momentum=momentum, kp=kp, dscale=dscale, act=act_name, rm=rm, rv=rv)
    return out


def bn_forward_bounds(f, u):
    x, mu, rstd, xhat, pre, g = f["x"], f["mean"], f["rstd"], f["xhat"], f["pre"], f["gamma"]
    rows = x.shape[0]
    b = {}
    if f["training"]:
        emu = C_COL * U32 * x.abs().sum(0) / rows + U32 * mu.abs()
        dd = (x - mu).abs()
        ed = emu + U32 * dd
        evar = (2 * (dd * ed).sum(0) + (ed * ed).sum(0) + C_COL * U32 * (dd * dd).sum(0)) / rows
        m = f["momentum"]
        b["save_mean"] = emu + TINY
        b["running_mean"] = m * emu + 4 * U32 * ((1 - m) * f["rm"].abs() + m * mu.abs()) + TINY
        r1 = rows / (rows - 1) if rows > 1 else 1.0
        b["running_var"] = m * evar * r1 + 4 * U32 * ((1 - m) * f["rv"].abs() + m * f["var"] * r1) + TINY
    else:
        emu = torch.zeros_like(mu)
        ed = U32 * (x - mu).abs()
        evar = torch.zeros_like(mu)
        b["save_mean"] = TINY
    erstd = rstd * (0.5 * evar / (f["var"] + f["eps"]) + 4 * U32)
    b["save_rstd"] = erstd + TINY
    epre = g.abs() * (ed * rstd + (x - mu).abs() * erstd) + C_EW * U32 * ((xhat * g).abs() + pre.abs())
    b["y_pre"] = epre + u * pre.abs() + TINY
    # the activation reads pre as stored (bf16 rounding) or un-rounded; the bf16 tanh is tanh.approx
    ein = epre + u * pre.abs()
    a = f["a"]
    if f["act"] == "tanh":
        ea = (1.0 - a * a) * ein + (E_TANH_APPROX if u == U_BF16 else 4 * U32) * a.abs()
    else:  # relu / none: 1-Lipschitz
        ea = ein
    sc = f["kp"] * f["dscale"] if f["kp"] is not None else 1.0
    b["y"] = (ea * sc + U32 * f["y"].abs()) + u * f["y"].abs() + TINY
    return b


def bn_backward(dy, x, y_pre, gamma, save_mean, save_rstd, *, act_name="none", kp=None, dscale=1.0):
    """g = dropout_bwd(dy) act'(y_pre) (y_pre as stored); xhat from the saved statistics;
    dx = gamma rstd (g - mean_rows(g) - xhat mean_rows(g xhat)); dgamma += sum_rows g xhat; dbeta += sum_rows g."""
    dy, x, gamma = dy.to(F64), x.to(F64), gamma.to(F64)
    mu, rstd = save_mean.to(F64), save_rstd.to(F64)
    rows = x.shape[0]
    gd = dy * kp * dscale if kp is not None else dy
    ad = act_grad(y_pre, act_name) if act_name != "none" else torch.ones_like(dy)
    g = gd * ad
    xhat = (x - mu) * rstd
    sg, sgx = g.sum(0), (g * xhat).sum(0)
    dx = gamma * rstd * (g - sg / rows - xhat * sgx / rows)
    return dict(gd=gd, ad=ad, g=g, xhat=xhat, sg=sg, sgx=sgx, dx=dx, dgamma=sgx, dbeta=sg, gamma=gamma, rstd=rstd,
                act=act_name, y_pre=None if y_pre is None else y_pre.to(F64))


def bn_backward_bounds(b, u):
    g, xhat, gamma, rstd = b["g"], b["xhat"], b["gamma"], b["rstd"]
    rows = g.shape[0]
    if b["act"] == "tanh":  # the bf16 vector kernel evaluates tanh(y_pre) with tanh.approx
        t = torch.tanh(b["y_pre"]).abs()
        ead = 2 * t * t * (E_TANH_APPROX if u == U_BF16 else 4 * U32) + 4 * U32
    else:
        ead = torch.zeros_like(g)
    eg = b["gd"].abs() * ead + 2 * U32 * g.abs()
    exh = 3 * U32 * xhat.abs()
    esg = C_COL * U32 * g.abs().sum(0) + eg.sum(0)
    esgx = C_COL * U32 * (g * xhat).abs().sum(0) + (eg * xhat.abs() + g.abs() * exh).sum(0)
    inner = g.abs() + b["sg"].abs() / rows + (xhat * b["sgx"]).abs() / rows
    edx = (gamma * rstd).abs() * (eg + esg / rows + exh * b["sgx"].abs() / rows + xhat.abs() * esgx / rows
                                  + C_EW * U32 * inner)
    return dict(dx=edx + u * b["dx"].abs() + TINY, dgamma=esgx + TINY, dbeta=esg + TINY)


# ============================================================================================ posenc
def posenc_forward(pe, alpha, T, *, tokens=None, emb=None, x=None, kp=None, dscale=1.0, u=U32):
    """y[b, t] = dropout((E[tokens[b, t]] or x[b, t]) + alpha pe[t]); only the first T rows of pe are read."""
    base = emb.to(F64)[tokens] if tokens is not None else x.to(F64)
    v = base + float(alpha) * pe.to(F64)[:T][None]
    y = v * kp * dscale if kp is not None else v
    bnd = C_EW * U32 * (base.abs() + abs(float(alpha)) * pe.to(F64)[:T][None].abs())
    if kp is not None:
        bnd = bnd * kp * dscale
    return y, bnd + u * y.abs() + TINY


def posenc_backward(dy, pe, T, *, tokens=None, padding_idx=-1, n_emb=0, kp=None, dscale=1.0):
    """g = dropout_bwd(dy); dx = g; demb[tok] += g[b, t] for every position whose token != padding_idx (repeats add);
    dalpha += sum g * pe[t]. Returns values and bounds."""
    dy = dy.to(F64)
    g = dy * kp * dscale if kp is not None else dy
    C = dy.shape[-1]
    p = pe.to(F64)[:T][None]
    out = dict(dx=g, dalpha=(g * p).sum(), b_dx=U32 * g.abs() + TINY,
               b_dalpha=C_GRID * U32 * (g * p).abs().sum() + TINY)
    if tokens is not None:
        use = (tokens != padding_idx).reshape(-1)
        tok = tokens.reshape(-1)[use]
        gg = g.reshape(-1, C)[use]
        out["demb"] = torch.zeros(n_emb, C, dtype=F64).index_add_(0, tok, gg)
        out["b_demb"] = C_COL * U32 * torch.zeros(n_emb, C, dtype=F64).index_add_(0, tok, gg.abs()) + TINY
    return out


# ============================================================================================ colsum, sumsq
def colsum(x, group_rows):
    """out[g][n] = sum of rows [g group_rows, min((g + 1) group_rows, rows)) of x (group_rows <= 0: one group)."""
    x = x.to(F64)
    rows = x.shape[0]
    gr = group_rows if group_rows > 0 else rows
    groups = (rows + gr - 1) // gr
    out = torch.stack([x[g * gr:(g + 1) * gr].sum(0) for g in range(groups)])
    bnd = C_COL * U32 * torch.stack([x[g * gr:(g + 1) * gr].abs().sum(0) for g in range(groups)]) + TINY
    return out, bnd


def sumsq(x):
    x = x.to(F64)
    s = (x * x).sum()
    return s, C_GRID * U32 * s + TINY


# ============================================================================================ Adam
def adam_step(p, g, m, v, *, lr, beta1, beta2, eps, weight_decay, step, grad_norm_sq, max_norm, grad_mul):
    """One update of fairseq/optim/adam.py:Adam.step after fairseq's clip_grad_norm_ on the grad_mul-scaled
    gradient: coef = min(max_norm / (sqrt(gn2) grad_mul + 1e-6), 1) (no clip when max_norm <= 0); g' = g grad_mul
    coef; m = b1 m + (1 - b1) g'; v = b2 v + (1 - b2) g'^2; p -= wd lr p; p -= lr sqrt(1 - b2^t) / (1 - b1^t) *
    m / (sqrt(v) + eps). A non-finite grad_norm_sq: nothing changes. Hyper-parameters are taken as the fp32 values
    the kernel receives. Returns dict(p, m, v, coef, step_size)."""
    p, g, m, v = (t.to(F64) for t in (p, g, m, v))
    lr, b1, b2, eps, wd, gm, mn = (f32(t) for t in (lr, beta1, beta2, eps, weight_decay, grad_mul, max_norm))
    gn2 = f32(grad_norm_sq)
    if not math.isfinite(gn2):
        return dict(p=p, m=m, v=v, coef=0.0, step_size=0.0, skipped=True)
    coef = 1.0
    if mn > 0:
        coef = min(mn / (math.sqrt(gn2) * gm + 1e-6), 1.0)
    gs = g * gm * coef
    m = b1 * m + (1 - b1) * gs
    v = b2 * v + (1 - b2) * gs * gs
    step_size = lr * math.sqrt(1 - b2 ** step) / (1 - b1 ** step)
    if wd != 0:
        p = p - wd * lr * p
    p = p - step_size * m / (torch.sqrt(v) + eps)
    return dict(p=p, m=m, v=v, coef=coef, step_size=step_size, skipped=False, gs=gs)


def adam_bounds(before, after, *, lr, beta1, beta2, eps, weight_decay, step, device_step=False):
    """Bounds of one kernel update started from the same (fp32) state `before` = (p, m, v). fp32 arithmetic on every
    operation; the device computes the bias correction with powf (a few ulps of b^t, amplified by 1 - b^t) when the
    step count comes from step_dev."""
    p0, m0, v0 = (t.to(F64) for t in before)
    lr, b1, b2, eps, wd = (f32(t) for t in (lr, beta1, beta2, eps, weight_decay))
    gs = after["gs"]
    em = C_EW * U32 * (b1 * m0.abs() + (1 - b1) * gs.abs() + after["m"].abs())
    ev = C_EW * U32 * (b2 * v0 + (1 - b2) * gs * gs + after["v"])
    sq = torch.sqrt(after["v"])
    den = sq + eps
    ss, am = after["step_size"], after["m"].abs()
    rel_ss = C_EW * U32
    if device_step:
        rel_ss += C_EW * U32 * (b1 ** step / (1 - b1 ** step) + 0.5 * b2 ** step / (1 - b2 ** step))
    # p -= ss m / (sqrt(v) + eps): errors of ss, m, v (through sqrt: ev / (2 sqrt v)) and of the operations
    eupd = ss / den * (em + am * (rel_ss + C_EW * U32) + am * torch.minimum(ev / (2 * sq.clamp_min(TINY)), sq) / den)
    ep = eupd + C_EW * U32 * (p0.abs() + wd * lr * p0.abs() + after["p"].abs())
    return dict(p=ep + TINY, m=em + TINY, v=ev + TINY)
