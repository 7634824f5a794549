"""fp64 statement of the loss entry points of include/speecht5_b200.h -- CTC (st5_ctc_loss), the TTS criterion
(st5_tts_loss_fwd / _bwd, st5_guided_attn_fwd / _bwd) and the speaker head (st5_l2norm_rows_fwd / _bwd,
st5_margin_ce_fwd / _bwd, st5_time_mean_fwd / _bwd) -- and elementwise error bounds for the kernels that implement them.
CPU only; no import of speecht5_b200.

Inputs are fp64 copies of exactly the values a kernel reads; fp32 hyper-parameters enter as the fp32 the kernel gets.
Bounds follow tests/rowops_ref.py: unit roundoff times fp64 magnitudes of the same operands, every fp32 reduction
bounded by (depth) * 2^-24 * sum |terms| with the depth read off the kernel's summation structure.

Device intrinsics (CUDA C Programming Guide, intrinsic functions): __expf(x) is within 2 + floor(1.173 |x|) ulp;
__logf(x) within 2^-21.41 absolute on [0.5, 2] and 3 ulp elsewhere; logf, log1pf, sqrtf, expf within 1-2 ulp.

CTC lattice bound. alpha_t(s) = lp_t(s) + lse2(lse2(alpha_{t-1}(s), alpha_{t-1}(s-1)), alpha_{t-1}(s-2)) in fp32 log
space. lse is 1-Lipschitz in the max norm, and more precisely |lse(a + e) - lse(a)| <= lse(a + |e|) - lse(a), so the
inherited error of state (t, s) is the weighted log-sum-exp of its predecessors' error budgets delta(t-1, .). Each step
then adds its own roundings: the two lse2 results and the final add (u times their magnitudes), the emission error of
lp_t(s) (row log-sum-exp plus the subtraction), and C_STEP0 u for the inner __expf / log1pf / difference terms (the
difference d = |a - b| enters log1p(exp(-d)) with slope <= 1/2 and d e^-d <= 1/e). Beta is the mirror image. The
posterior exponent e = alpha + beta - lp + nll then carries delta_alpha + delta_beta + the lp error + delta_nll plus
the rounding of the four-term sum, u (|alpha| + |beta| + |lp| + |nll|) per addition; each term exp(e) has relative error
expm1(delta_e) plus __expf's ulp error. Terms with e <= -80 are dropped by the kernel: at most S e^-80 per row."""
import math

import torch

from rowops_ref import F64, TINY, U32, U_BF16, check, exceeds, f32  # noqa: F401  (re-exported for the tests)

# __expf: 2 + floor(1.173 |x|) ulp; __logf: 2^-21.41 absolute on [0.5, 2], else 3 ulp
EXPF_ULP0, EXPF_ULP1 = 2.0, 1.173
LOGF_ABS, LOGF_ULP = 2.0 ** -21.41, 3.0
# per lattice step: two lse2 inner terms (__expf <= 2.5 u absolute after the log1p, log1pf 1 ulp of <= log 2, the
# difference <= 0.3 u) and slack for the constant parts of the adds
C_STEP0 = 8.0
# posterior exponent alpha + beta - lp + nll: three fp32 additions, each rounded to u of a partial sum bounded by the
# sum of the four magnitudes
C_POST = 3.0
# TTS / guided reductions: the in-lane chain, 5 shuffle levels, the 8-warp CTA sum, the 8-level tree of the fixed-order
# sum, plus the multiplications that form the means (a few u)
C_TREE = 5 + 8 + 8 + 4
# speaker-head block sums: 5 shuffle levels + the 8 warp partials added serially
C_BLOCK = 5 + 8


# ============================================================================================ CTC
def ctc_row_lse(x):
    """lse over the last dim of fp64 values x [..., V] and the error of m + __logf(sum __expf(x - m)) (warp per row:
    ceil(V / 32) terms per lane, a 5-level tree)."""
    V = x.shape[-1]
    m = x.max(-1, keepdim=True).values
    d = x - m
    e = torch.exp(d)
    s = e.sum(-1)
    ls = torch.log(s)
    lse = m[..., 0] + ls
    rel_s = U32 * (math.ceil(V / 32) + 5) + U32 * (e * (EXPF_ULP0 + (EXPF_ULP1 + 1) * d.abs())).sum(-1) / s
    err = 1.01 * rel_s + LOGF_ULP * U32 * ls.abs() + LOGF_ABS + U32 * lse.abs()
    return lse, err


def _ext(tg, blank):
    """Extended label sequence (blank, l1, blank, ..., lL, blank) and the skip mask (s odd, s >= 2, l'_s != l'_{s-2})."""
    L = len(tg)
    S = 2 * L + 1
    lab = torch.full((S,), blank, dtype=torch.long)
    lab[1::2] = tg
    skip = torch.zeros(S, dtype=torch.bool)
    if L > 1:
        skip[3::2] = tg[1:] != tg[:-1]
    return lab, skip


def _shift(v, k, fill):
    """v shifted right by k (k > 0) or left (k < 0) along the last dim, `fill` coming in."""
    out = torch.full_like(v, fill)
    if k > 0:
        out[k:] = v[:-k]
    else:
        out[:k] = v[-k:]
    return out


def _beta_skip(skip):
    """beta of s takes s + 2 exactly where alpha of s + 2 took s (l'_s != blank, l'_s != l'_{s+2})."""
    return _shift(skip, -2, False)


def _lse_stack(vals):
    return torch.logsumexp(torch.stack(vals), 0)


def _sweep(lp, lerr, skip, S, reverse):
    """alpha (reverse=False) or beta lattice [Tn, S] in fp64 and its error budget delta [Tn, S]."""
    Tn = lp.shape[0]
    NINF = -math.inf
    a = torch.full((Tn, S), NINF, dtype=F64)
    dl = torch.zeros((Tn, S), dtype=F64)
    d1 = 1 if not reverse else -1
    skip_here = skip if not reverse else _beta_skip(skip)
    steps = range(Tn) if not reverse else range(Tn - 1, -1, -1)
    prev = prevd = None
    for t in steps:
        if prev is None:
            init = torch.full((S,), NINF, dtype=F64)
            if not reverse:
                init[:2] = 0.0
            else:
                init[max(S - 2, 0):] = 0.0
            a[t] = init + lp[t]
            dl[t] = torch.where(torch.isfinite(a[t]), lerr[t], torch.zeros_like(lerr[t]))
        else:
            p1 = _shift(prev, d1, NINF)
            p2 = torch.where(skip_here, _shift(prev, 2 * d1, NINF), torch.full_like(prev, NINF))
            v1 = _lse_stack([prev, p1])
            v2 = _lse_stack([v1, p2])
            q = torch.where(torch.isfinite(prevd), prevd, torch.zeros_like(prevd))
            inh = _lse_stack([prev + q, _shift(prev + q, d1, NINF),
                              torch.where(skip_here, _shift(prev + q, 2 * d1, NINF), torch.full_like(prev, NINF))]) - v2
            a[t] = v2 + lp[t]
            fin = torch.isfinite(a[t])
            loc = U32 * (torch.nan_to_num(v1.abs(), posinf=0.0) + torch.nan_to_num(v2.abs(), posinf=0.0)
                         + torch.nan_to_num(a[t].abs(), posinf=0.0) + C_STEP0)
            dl[t] = torch.where(fin, torch.nan_to_num(inh, nan=0.0) + loc + lerr[t], torch.zeros_like(loc))
        prev, prevd = a[t], dl[t]
    return a, dl


def ctc(logits, targets, input_lengths, *, blank, zero_infinity, S_max):
    """logits [T, B, V] (fp64 of what the kernel reads), targets: list of B int64 label tensors, input_lengths: B ints.
    Returns dict(nll [B], grad [T, B, V], feasible [B]) and the bounds b_nll, b_grad. nll is +inf on an infeasible
    utterance (0 with zero_infinity); rows t >= min(T, input_lengths[b]) and infeasible utterances get zero gradient."""
    x = logits.to(F64)
    T, B, V = x.shape
    lse, lse_err = ctc_row_lse(x)                   # [T, B]
    nll = torch.zeros(B, dtype=F64)
    b_nll = torch.full((B,), TINY, dtype=F64)
    grad = torch.zeros(T, B, V, dtype=F64)
    b_grad = torch.full((T, B, V), TINY, dtype=F64)
    feasible = torch.zeros(B, dtype=torch.bool)
    amax = 0.0
    for b in range(B):
        tg = targets[b].to(torch.long)
        S = 2 * len(tg) + 1
        Tn = min(T, int(input_lengths[b]))
        if Tn < 1 or S > S_max:
            nll[b] = 0.0 if zero_infinity else math.inf
            continue
        lab, skip = _ext(tg, blank)
        lp = x[:Tn, b][:, lab] - lse[:Tn, b, None]  # [Tn, S]
        lerr = lse_err[:Tn, b, None] + U32 * lp.abs()
        al, da = _sweep(lp, lerr, skip, S, False)
        be, db = _sweep(lp, lerr, skip, S, True)
        fin_idx = [S - 1, S - 2] if S >= 2 else [0]
        ll = torch.logsumexp(al[Tn - 1, fin_idx], 0)
        if not math.isfinite(float(ll)):
            nll[b] = 0.0 if zero_infinity else math.inf
            continue
        feasible[b] = True
        nb = -float(ll)
        q = da[Tn - 1, fin_idx]
        dn = float(torch.logsumexp(al[Tn - 1, fin_idx] + q, 0) - ll) + U32 * (abs(nb) + C_STEP0)
        nll[b] = nb
        b_nll[b] = dn + TINY
        amax = max(amax, float(torch.nan_to_num(al.abs(), posinf=0.0).max()))
        e = al + be - lp + nb                         # [Tn, S]
        pm = torch.exp(e)
        fin = torch.isfinite(e)
        de = (da + db + lerr + dn
              + C_POST * U32 * (al.abs() + be.abs() + lp.abs() + abs(nb)))
        de = torch.where(fin, de, torch.zeros_like(de))
        e_term = torch.where(fin, pm * (torch.expm1(de) + U32 * (EXPF_ULP0 + EXPF_ULP1 * e.abs())),
                             torch.zeros_like(pm))
        pm = torch.where(fin, pm, torch.zeros_like(pm))
        post = torch.zeros(Tn, V, dtype=F64).index_add_(1, lab, pm)
        epost = torch.zeros(Tn, V, dtype=F64).index_add_(1, lab, e_term)
        # summation depth per symbol: the blank's per-lane chains + 5 shuffles + 1; a label's atomics: its state count
        cnt = torch.zeros(V, dtype=F64).index_add_(0, lab, torch.ones(S, dtype=F64))
        depth = cnt + 1.0
        depth[blank] = math.ceil(S / 32) + 5 + 1
        xs = x[:Tn, b]
        d = xs - lse[:Tn, b, None]
        sm = torch.exp(d)
        g = sm - post
        esm = sm * (lse_err[:Tn, b, None] + U32 * (EXPF_ULP0 + (EXPF_ULP1 + 1) * d.abs()))
        grad[:Tn, b] = g
        b_grad[:Tn, b] = (esm + epost + U32 * depth * post + cnt * math.exp(-80.0) + U32 * g.abs() + TINY)
    return dict(nll=nll, grad=grad, feasible=feasible, b_nll=b_nll, b_grad=b_grad, amax=amax)


# ============================================================================================ TTS loss
def _softplus(x):
    return torch.clamp_min(x, 0) + torch.log1p(torch.exp(-x.abs()))


def tts_valid(olens, L, r):
    """valid[b, l] = l < ol[b] = olens[b] - olens[b] % r (text_to_speech_loss.py:164)."""
    ol = torch.tensor([int(o) - int(o) % r for o in olens])
    return torch.arange(L)[None, :] < ol[:, None], ol


def _stop_target(labels, ol, r):
    """The stop labels with 1 at the last valid frame ol - 1 when r > 1 (the scatter of text_to_speech_loss.py:168)."""
    t = labels.clone()
    if r > 1:
        for b in range(t.shape[0]):
            if 1 <= ol[b] <= t.shape[1]:
                t[b, ol[b] - 1] = 1.0
    return t


def _bce_terms(x, t, pw):
    """BCEWithLogits with pos_weight on the positive term: pw t softplus(-x) + (1 - t) softplus(x)."""
    return pw * t * _softplus(-x) + (1 - t) * _softplus(x)


def tts_loss(after, before, logits, ys, labels, olens, *, r, pos_weight, g=(1.0, 1.0, 1.0)):
    """after / before [B, L, D], logits [B, L], ys [B, >= L, D], labels [B, >= L] (only l < L is used). Returns the
    three means (l1, l2, bce), n (valid frames) and the gradients for upstream g, with elementwise bounds."""
    a, bf, x = after.to(F64), before.to(F64), logits.to(F64)
    B, L, D = a.shape
    y = ys.to(F64)[:, :L]
    valid, ol = tts_valid(olens, L, r)
    t = _stop_target(labels.to(F64)[:, :L], ol, r)
    pw = f32(pos_weight)
    v = valid.to(F64)
    n = float(v.sum())
    da, db = (a - y) * v[..., None], (bf - y) * v[..., None]
    da = torch.nan_to_num(da, nan=0.0)
    db = torch.nan_to_num(db, nan=0.0)
    s1 = (da.abs() + db.abs()).sum()
    s2 = (da * da + db * db).sum()
    xz = torch.where(valid, x, torch.zeros_like(x))
    tz = torch.where(valid, t, torch.zeros_like(t))
    terms = _bce_terms(xz, tz, pw) * v
    sb = terms.sum()
    inv = 1.0 / n if n > 0 else 0.0
    out = torch.stack([s1 * inv / D, s2 * inv / D, sb * inv])
    nblk = math.ceil(B * L / 8)
    depth = math.ceil(2 * D / 32) + 8 + C_TREE + math.ceil(nblk / 256)
    e1 = (depth + 2) * U32 * s1
    e2 = (depth + 3) * U32 * s2
    # softplus = max(x, 0) + log1pf(__expf(-|x|)): <= 2.5 u from __expf after the log1p, 1 ulp of log1pf, u |sp|
    # from the add; then the weight products and the two-term sum (3 u |term|)
    eb = depth * U32 * terms.abs().sum() + ((4 * U32 * (pw * tz + 1 - tz)) * v).sum() + 4 * U32 * terms.abs().sum()
    b_out = torch.stack([e1 * inv / D, e2 * inv / D, eb * inv]) + 4 * U32 * out.abs() + TINY
    # gradients
    g0, g1, g2 = (float(v_) for v_ in g)
    k1, k2 = g0 * inv / D, 2 * g1 * inv / D

    def grad1(d):
        return (torch.sign(d) * k1 + k2 * d) * v[..., None]

    d_after, d_before = grad1(da), grad1(db)
    sg = torch.sigmoid(xz)
    c = pw * tz + 1 - tz
    d_logits = g2 * inv * (sg * c - pw * tz) * v

    def egrad(d):
        return (6 * U32 * (abs(k1) + (k2 * d).abs()) + 2 * abs(k2) * U32 * d.abs()) * v[..., None] + TINY

    e_lg = abs(g2 * inv) * (c * sg * U32 * (5 + EXPF_ULP1 * xz.abs()) + U32 * (c * sg + pw * tz)) * v \
        + 4 * U32 * d_logits.abs() + TINY
    return dict(out=out, n=n, b_out=b_out, d_after=d_after, d_before=d_before, d_logits=d_logits,
                b_d_after=egrad(da), b_d_before=egrad(db), b_d_logits=e_lg, valid=valid, target=t)


# ============================================================================================ guided attention
def _ol_w(olen, r):
    """The decoder-step length W divides by: olens[b] / r (text_to_speech_loss.py:163), not clamped to T_out."""
    return int(olen) // r


def guided_w(il_u, ol_u, ol_region, T_out, T_in, sigma):
    """W [T_out, T_in] = 1 - exp(-(ti / il - to / ol)^2 / (2 sigma^2)) with the unclamped lengths, its error bound as
    the kernel evaluates it (fp32 to / ol, 1 / il, ti * (1 / il), __expf), and the region to < min(T_out, ol_region),
    ti < min(T_in, il_u)."""
    sig = f32(sigma)
    k = 1.0 / (2 * sig * sig)
    to = torch.arange(T_out, dtype=F64)[:, None]
    ti = torch.arange(T_in, dtype=F64)[None, :]
    il_c, ol_c = min(T_in, il_u), min(T_out, ol_region)
    region = (to < ol_c) & (ti < il_c)
    if il_u <= 0 or ol_u <= 0:
        z = torch.zeros(T_out, T_in, dtype=F64)
        return z, z + TINY, region
    gx = to / ol_u
    fx = ti / il_u
    dlt = fx - gx
    q = dlt * dlt * k
    E = torch.exp(-q)
    W = 1.0 - E
    e_d = 3 * U32 * (fx.abs() + gx.abs() + dlt.abs())
    e_q = 2 * dlt.abs() * e_d * k + 6 * U32 * q
    e_W = E * (e_q + U32 * (EXPF_ULP0 + EXPF_ULP1 * q)) + U32 * W.abs() + U32
    return W, e_W, region


def guided(att, ilens, olens, *, r, heads, sigma, alpha, g=1.0):
    """att: list of n_layers tensors [B, H, T_out, T_in] (only the valid region is read). Returns out, gsum0, gsum1 and
    datt (list, [B, heads, T_out, T_in], zero outside the region) with bounds."""
    nl = len(att)
    B, H, T_out, T_in = att[0].shape
    al = f32(alpha)
    Ws, eWs, regs = [], [], []
    n = 0.0
    for b in range(B):
        ol_u, il_u = int(olens[b]) // r, int(ilens[b])
        W, eW, reg = guided_w(il_u, _ol_w(olens[b], r), ol_u, T_out, T_in, sigma)
        Ws.append(W)
        eWs.append(eW)
        regs.append(reg)
        n += min(T_out, ol_u) * min(T_in, il_u)
    n *= heads * nl
    W = torch.stack(Ws)[:, None]
    eW = torch.stack(eWs)[:, None]
    reg = torch.stack(regs)[:, None]
    s0, sa, se = 0.0, 0.0, 0.0
    for a in att:
        A = torch.where(reg, a.to(F64)[:, :heads], torch.zeros(1, dtype=F64))
        s0 += float((W * A).sum())
        sa += float((W * A).abs().sum())
        se += float((eW * A.abs()).sum())
    nrows = nl * B * heads * T_out
    depth = math.ceil(T_in / 32) + C_TREE + math.ceil(math.ceil(nrows / 8) / 256)
    e0 = depth * U32 * sa + se + TINY
    out = al * s0 / n if n > 0 else 0.0
    b_out = (abs(al) * e0 / n + 4 * U32 * abs(out) if n > 0 else 0.0) + TINY
    kk = g * al / n if n > 0 else 0.0
    datt = torch.where(reg, kk * W, torch.zeros(1, dtype=F64)).expand(B, heads, T_out, T_in)
    b_datt = torch.where(reg, abs(kk) * (eW + 3 * U32 * W.abs()), torch.zeros(1, dtype=F64)).expand(
        B, heads, T_out, T_in) + TINY
    return dict(out=out, b_out=b_out, gsum0=s0, b_gsum0=e0, gsum1=n, datt=datt, b_datt=b_datt, region=reg)


# ============================================================================================ speaker head
L2_EPS = 1e-12


def l2norm_fwd(x):
    """y = x / max(||x||, 1e-12), nrm = ||x|| per row of x [rows, E] (warp per row)."""
    x = x.to(F64)
    E = x.shape[1]
    ss = (x * x).sum(1)
    n = torch.sqrt(ss)
    den = n.clamp_min(L2_EPS)
    y = x / den[:, None]
    depth = math.ceil(E / 32) + 5 + 1
    rel_n = 0.5 * depth * U32 + U32
    return dict(y=y, nrm=n, b_y=y.abs() * (rel_n * (n >= L2_EPS).to(F64)[:, None] + 3 * U32) + TINY,
                b_nrm=n * rel_n + TINY)


def l2norm_bwd(dy, y, nrm):
    """dx = (dy - y <dy, y>) / ||x||, or dy / 1e-12 on a clamped row (the dot product is skipped there)."""
    dy, y, nrm = dy.to(F64), y.to(F64), nrm.to(F64)
    E = dy.shape[1]
    clamped = nrm < L2_EPS
    dot = torch.where(clamped, torch.zeros_like(nrm), (dy * y).sum(1))
    inv = 1.0 / nrm.clamp_min(L2_EPS)
    inner = dy - y * dot[:, None]
    dx = inner * inv[:, None]
    depth = math.ceil(E / 32) + 5 + 1
    edot = depth * U32 * (dy * y).abs().sum(1) * (~clamped).to(F64)
    e = inv[:, None] * (y.abs() * edot[:, None] + 2 * U32 * (dy.abs() + (y * dot[:, None]).abs())) \
        + 2 * U32 * dx.abs()
    return dx, e + TINY


def margin_consts(mode, scale, margin):
    """The fp32 constants the launcher derives on the host (cosf / sinf of the fp32 margin, pi as an fp32)."""
    m = f32(margin)
    pi_f = f32(math.pi)
    return dict(mode=mode, s=f32(scale), m=m, cos_m=f32(math.cos(m)), sin_m=f32(math.sin(m)),
                th=f32(math.cos(f32(pi_f - m))), mm=f32(f32(math.sin(f32(pi_f - m))) * m))


def margin_logits(x, mt, c, easy):
    """z [B, N] from cosines x and the margin column mt (None: plain logits) with constants c; error bound; slope
    dz/dx; its error bound."""
    x = x.to(F64)
    B, N = x.shape
    if mt is None:
        return x, torch.full_like(x, TINY), torch.ones_like(x), torch.zeros_like(x)
    s = c["s"]
    z = s * x
    ez = U32 * z.abs()
    slope = torch.full_like(x, s)
    eslope = torch.zeros_like(x)
    rows = torch.arange(B)
    xt = x[rows, mt]
    if c["mode"] == 1:  # AM
        zt = s * (xt - c["m"])
        ezt = 2 * U32 * (s * xt).abs() + 2 * U32 * abs(s * c["m"]) + U32 * zt.abs()
        st, est = torch.full_like(xt, s), torch.zeros_like(xt)
    else:  # AAM
        q = 1.0 - xt * xt
        sine = torch.sqrt(q.clamp(0, 1))
        phi = xt * c["cos_m"] - sine * c["sin_m"]
        keep = xt > 0 if easy else xt > c["th"]
        other = xt if easy else xt - c["mm"]
        zt = s * torch.where(keep, phi, other)
        eq = 2 * U32 * (xt * xt + q.abs())
        esine = torch.minimum(eq / (2 * sine.clamp_min(TINY)), eq.sqrt()) + U32 * sine
        ephi = 2 * U32 * (xt * c["cos_m"]).abs() + esine * c["sin_m"] + 2 * U32 * sine * c["sin_m"] + U32 * phi.abs()
        eoth = 0 if easy else 2 * U32 * (xt.abs() + c["mm"])
        ezt = s * torch.where(keep, ephi, eoth + torch.zeros_like(ephi)) + U32 * zt.abs()
        ds = torch.where((q >= 0) & (q <= 1) & (sine > 0), -xt / sine.clamp_min(TINY), torch.zeros_like(xt))
        st = s * torch.where(keep, c["cos_m"] - ds * c["sin_m"], torch.ones_like(xt))
        eds = torch.where(sine > 0, ds.abs() * (esine / sine.clamp_min(TINY) + 2 * U32), torch.zeros_like(xt))
        est = s * torch.where(keep, eds * c["sin_m"] + 3 * U32 * (c["cos_m"] + (ds * c["sin_m"]).abs()),
                              torch.zeros_like(xt))
    z[rows, mt], ez[rows, mt] = zt, ezt
    slope[rows, mt], eslope[rows, mt] = st, est
    return z, ez + TINY, slope, eslope


def margin_ce_fwd(x, mt, target, *, mode, scale, margin, easy, eps, ignore_index):
    """Forward of st5_margin_ce_fwd: z, and with target: per-row loss, nll, correct, valid, lse (bounded)."""
    c = margin_consts(mode, scale, margin)
    z, ez, slope, eslope = margin_logits(x, mt, c, easy)
    B, N = z.shape
    out = dict(z=z, b_z=ez, slope=slope, b_slope=eslope, consts=c)
    if target is None:
        return out
    mx = z.max(1, keepdim=True).values
    d = z - mx
    e = torch.exp(d)
    se = e.sum(1)
    lse = mx[:, 0] + torch.log(se)
    depth = math.ceil(N / 256) + C_BLOCK + 1
    elz = ez.max(1).values
    e_lse = (depth * U32 + U32 * (e * (EXPF_ULP0 + (EXPF_ULP1 + 1) * d.abs())).sum(1) / se) * 1.01 \
        + 2 * U32 * torch.log(se).abs() + U32 * lse.abs() + 2 * elz
    eps_f = f32(eps)
    eps_i = eps_f / (N - 1)
    tt = torch.as_tensor(target).to(torch.long)
    valid = tt != ignore_index
    inb = (tt >= 0) & (tt < N)
    tc = tt.clamp(0, N - 1)
    rows = torch.arange(B)
    zt = z[rows, tc]
    nll = lse - zt
    sz = z.sum(1)
    smooth = N * lse - sz
    loss = (1 - eps_f - eps_i) * nll + eps_i * smooth
    e_nll = e_lse + ez[rows, tc] + U32 * nll.abs()
    e_sz = depth * U32 * z.abs().sum(1) + ez.sum(1)
    e_sm = N * e_lse + U32 * N * lse.abs() + e_sz + U32 * smooth.abs()
    e_loss = (1 - eps_f - eps_i) * e_nll + eps_i * e_sm + 4 * U32 * ((1 - eps_f - eps_i) * nll.abs()
                                                                     + eps_i * smooth.abs()) + 2 * U32 * abs(eps_f) \
        * (nll.abs() + smooth.abs() / (N - 1))
    am = torch.argmax(z, 1)  # first maximum (torch.argmax)
    srt = torch.sort(z, 1, descending=True).values
    ambiguous = (srt[:, 0] - srt[:, 1] <= 2 * elz) & (srt[:, 0] != srt[:, 1])
    zero = torch.zeros(B, dtype=F64)
    nan = torch.full((B,), math.nan, dtype=F64)
    loss = torch.where(valid, torch.where(inb, loss, nan), zero)
    nll = torch.where(valid, torch.where(inb, nll, nan), zero)
    out.update(lse=lse, b_lse=e_lse + TINY, loss=loss, b_loss=torch.where(valid, e_loss, zero) + TINY, nll=nll,
               b_nll=torch.where(valid, e_nll, zero) + TINY, correct=((am == tt) & valid).to(F64),
               valid=valid.to(F64), ambiguous=ambiguous, eps_i=eps_i)
    return out


def margin_ce_bwd(f, target, *, eps, ignore_index, gstat=None, dz_in=None):
    """dx = dz * dz/dx from the forward's statement f; dz from (loss, nll) with gstat = (ga, gn), or given (dz_in)."""
    z, slope = f["z"], f["slope"]
    B, N = z.shape
    if dz_in is not None:
        dz = dz_in.to(F64)
        edz = torch.zeros_like(dz)
    else:
        ga, gn = (f32(v) for v in gstat)
        eps_f, eps_i = f32(eps), f["eps_i"]
        tt = torch.as_tensor(target).to(torch.long)
        valid = (tt != ignore_index).to(F64)[:, None]
        dd = z - f["lse"][:, None]
        p = torch.exp(dd)
        hit = torch.nn.functional.one_hot(tt.clamp(0, N - 1), N).to(F64)
        w1 = 1 - eps_f - eps_i
        dz = (ga * (w1 * (p - hit) + eps_i * (N * p - 1)) + gn * (p - hit)) * valid
        ep = p * ((f["b_z"] + f["b_lse"][:, None] + U32 * dd.abs()) * 1.01 + U32 * (EXPF_ULP0 + EXPF_ULP1 * dd.abs()))
        edz = ((abs(ga) * (abs(w1) + eps_i * N) + abs(gn)) * ep
               + 8 * U32 * (abs(ga) * (abs(w1) * (p + hit) + eps_i * (N * p + 1)) + abs(gn) * (p + hit))) * valid
    dx = dz * slope
    edx = edz * slope.abs() + dz.abs() * f["b_slope"] + U32 * dx.abs() + TINY
    return dx, edx


def time_mean_fwd(x, u):
    """y[b, c] = mean over all T frames of x [B, T, C]; per thread T / 8 frames, then 8 partials in order."""
    x = x.to(F64)
    T = x.shape[1]
    y = x.mean(1)
    depth = math.ceil(T / 8) + 8 + 1
    return y, depth * U32 * x.abs().sum(1) / T + U32 * y.abs() + u * y.abs() + TINY


def time_mean_bwd(dy, T, u):
    dx = (dy.to(F64) / T)[:, None, :].expand(dy.shape[0], T, dy.shape[1])
    return dx, U32 * dx.abs() + u * dx.abs() + TINY
