"""fp64 statement of the attention contract of include/speecht5_b200.h (st5_attn_args and the fused / streaming /
tensor-core entry points), and elementwise error bounds for the kernels that implement it. CPU only; no import of
speecht5_b200.

Layout: q [B, H, Tq, 64], k / v [B, H, Tk, 64] (fp64 copies of exactly the values the kernel reads: the bf16 operands,
and the bf16 copy of the position table for the wgmma kernels / the fp32 table for the row kernels).

  s[i, j]  = scale * q_i . (k_j + pe[clamp(i - j, -maxpos, maxpos - 1) + maxpos])       (pe optional)
  masks    : causal (j > i), key_pad[b, j] != 0  ->  -inf
  P        = softmax_j(s);  e = exp(s - rowmax) (0 on masked keys), l = sum_j e, lse = log l + rowmax
  Pd       = P * keep * drop_scale  (keep: dropout_ref.attn_keep)
  out      = Pd @ v
  backward : dPd = dO v^T;  dP = dPd * keep * drop_scale + dP_ext;  delta = sum_j P dP  (= dO . out + sum_j P dP_ext)
             dS = P (dP - delta);  dQ = scale (dS k + dQP pe);  dK = scale dS^T q;  dV = Pd^T dO
             dQP[i, r] = sum_{j : idx(i, j) = r} dS[i, j];  dPE[r] = scale sum_{b, h, i} dQP[b, h, i, r] q_i

Bounds (`bounds`) are built like tests/test_gemm_contract_gpu.py: a constant times a unit roundoff times an fp64
magnitude product of the same operands, elementwise. `u` is the unit of the narrowest storage step (2^-8 for bf16
operands / outputs, ~2^-22 for the fp32 row kernels); score rounding (fp32 accumulation of 64 products, exponent
argument) is carried separately as a relative error of P."""
import math

import numpy as np
import torch

import dropout_ref as D

F64 = torch.float64
U_BF16 = 2.0 ** -8
U_F32 = 2.0 ** -22
TINY = 2.0 ** -60
# Bound constants, set on an H100 80GB HBM3 (400 W power limit). Largest err / bound observed over
# tests/test_attention_contract_gpu.py: 0.73 (st5_attn_fused_bwd dV) for the bf16 kernels with C_BF16; 0.03 for the
# fp32 row kernels with C_F32. The pure bf16-rounding terms (u |ref|) reach 0.99 by construction: round-to-nearest
# bf16 is within 2^-8 |x|.
C_BF16 = 2.0
C_F32 = 8.0


def _rows(Tq, rows):
    return torch.arange(Tq) if rows is None else torch.as_tensor(rows)


def rel_index(Tq, Tk, maxpos, rows=None):
    """[Tq, Tk] table row of (i, j): clamp(i - j, -maxpos, maxpos - 1) + maxpos. rows: absolute query indices."""
    d = _rows(Tq, rows)[:, None] - torch.arange(Tk)[None, :]
    return d.clamp(-maxpos, maxpos - 1) + maxpos


def valid_mask(B, Tq, Tk, causal=False, key_pad=None, rows=None):
    """[B, 1, Tq, Tk] bool: key j takes part in row i."""
    ok = torch.ones(B, 1, Tq, Tk, dtype=torch.bool)
    if causal:
        ok &= (torch.arange(Tk)[None, :] <= _rows(Tq, rows)[:, None])[None, None]
    if key_pad is not None:
        ok &= ~key_pad.bool()[:, None, None, :]
    return ok


def keep_mask(B, H, Tq, Tk, drop_p, seed, offset):
    if drop_p <= 0:
        return torch.ones(B, H, Tq, Tk, dtype=torch.bool)
    return torch.from_numpy(D.attn_keep(seed, offset, drop_p, B, H, Tq, Tk))


def _qpe(q, pe, Tk, maxpos, rows=None):
    """q_i . pe[idx(i, j)] as [B, H, Tq, Tk]: QP = q pe^T gathered along the table axis."""
    Tq = q.shape[2]
    qp = q @ pe.T  # [B, H, Tq, 2 maxpos]
    idx = rel_index(Tq, Tk, maxpos, rows).expand(q.shape[0], q.shape[1], Tq, Tk)
    return torch.gather(qp, 3, idx)


def forward(q, k, v, *, scale, pe=None, maxpos=0, causal=False, key_pad=None, drop_p=0.0, seed=0, offset=0,
            keep=None, rows=None):
    """Every forward quantity of the contract, fp64. Returns a dict. rows (optional): the absolute indices of the
    query rows q holds (a subset of a longer sequence; then pass `keep` too if there is dropout)."""
    q, k, v = q.to(F64), k.to(F64), v.to(F64)
    B, H, Tq, _ = q.shape
    Tk = k.shape[2]
    s = scale * (q @ k.transpose(-1, -2))
    if pe is not None:
        s = s + scale * _qpe(q, pe.to(F64), Tk, maxpos, rows)
    ok = valid_mask(B, Tq, Tk, causal, key_pad, rows).expand(B, H, Tq, Tk)
    s = s.masked_fill(~ok, -math.inf)
    m = s.amax(-1, keepdim=True)
    e = torch.exp(s - m).masked_fill(~ok, 0.0)
    l = e.sum(-1, keepdim=True)
    P = e / l
    if keep is None:
        keep = keep_mask(B, H, Tq, Tk, drop_p, seed, offset)
    dscale = D.drop_scale(drop_p)
    Pd = P * keep * dscale
    out = Pd @ v
    return dict(q=q, k=k, v=v, pe=None if pe is None else pe.to(F64), scale=scale, maxpos=maxpos, rows=rows, ok=ok,
                s=s, m=m,
                e=e, l=l, P=P, keep=keep, dscale=dscale, Pd=Pd, out=out, inv_l=(1.0 / l)[..., 0],
                lse=(torch.log(l) + m)[..., 0])


def scatter_qp(dS, maxpos):
    """dQP[.., i, r] = sum over keys j with idx(i, j) == r of dS[.., i, j]."""
    Tq, Tk = dS.shape[-2:]
    idx = rel_index(Tq, Tk, maxpos).expand(*dS.shape)
    out = torch.zeros(*dS.shape[:-1], 2 * maxpos, dtype=dS.dtype)
    return out.scatter_add_(-1, idx, dS)


def head_major(x):
    """[B, H, ...] -> [H, B, ...] (the row order of st5_attn_dqp_scatter with h_major)."""
    return x.transpose(0, 1).contiguous()


def backward(f, dO, dP_ext=None):
    """Every backward quantity of the contract, fp64; `f` from forward()."""
    dO = dO.to(F64)
    dPd = dO @ f["v"].transpose(-1, -2)
    dP = dPd * f["keep"] * f["dscale"]
    if dP_ext is not None:
        dP = dP + dP_ext.to(F64)
    dP = dP.masked_fill(~f["ok"], 0.0)  # (P is 0 there: the value does not reach dS)
    P = f["P"]
    delta = (P * dP).sum(-1)
    dS = P * (dP - delta[..., None])
    sc = f["scale"]
    g = dict(dO=dO, dPd=dPd, dP=dP, delta=delta, dS=dS)
    g["dQ_k"] = sc * (dS @ f["k"])  # the q.k part (st5_attn_fused_bwd with relative positions writes only this)
    g["dQ"] = g["dQ_k"]
    g["dK"] = sc * (dS.transpose(-1, -2) @ f["q"])
    g["dV"] = f["Pd"].transpose(-1, -2) @ dO
    if f["pe"] is not None:
        dQP = scatter_qp(dS, f["maxpos"])
        g["dQP"] = dQP
        g["dQ"] = g["dQ_k"] + sc * (dQP @ f["pe"])
        g["dPE"] = sc * torch.einsum("bhir,bhic->rc", dQP, f["q"])
    return g


def score_error(f, Cs):
    """Relative error of each exp(s - rowmax) from the fp32 score and exponent argument (see `bounds`)."""
    q, k, sc = f["q"], f["k"], f["scale"]
    aq, ak = q.abs(), k.abs()
    smag = sc * (aq @ ak.transpose(-1, -2))
    if f["pe"] is not None:
        smag = smag + sc * _qpe(aq, f["pe"].abs(), k.shape[2], f["maxpos"], f["rows"])
    s_abs = torch.where(f["ok"], f["s"].abs(), torch.zeros_like(smag))
    smag = torch.where(f["ok"], smag, torch.zeros_like(smag))
    return Cs * 2.0 ** -24 * (smag + s_abs + (smag + s_abs).amax(-1, keepdim=True) + 4.0)


def bounds(f, g=None, *, u, C, Cs=64.0):
    """Elementwise bounds, same shapes as the quantities. `u`: storage unit roundoff; `C`: constant set on the H100.

    Score error: fp32 accumulation of the 64-term dot products and of the exponent argument, relative to the magnitude
    Smag = scale |q| . (|k| + |pe|). P inherits it twice (its own score and the row's normaliser):
    EP = P * Cs 2^-24 (Smag_ij + |s_ij| + max_j (Smag + |s|) + 4)."""
    q, k, v, sc = f["q"], f["k"], f["v"], f["scale"]
    aq, ak, av = q.abs(), k.abs(), v.abs()
    es = score_error(f, Cs)
    P, Pd = f["P"], f["Pd"]
    EP = P * es
    EPd = EP * f["keep"] * f["dscale"]
    b = {}
    b["P"] = EP + u * P + TINY                       # returned probabilities (fp32: u = U_F32)
    b["e"] = f["e"] * (es + u) + TINY                # psave: exp(s - max), bf16
    b["inv_l"] = f["inv_l"] * (es.amax(-1) + u)      # 1 / rowsum (fp32 store)
    b["lse"] = es.amax(-1) + u * f["lse"].abs() + TINY
    b["out"] = C * u * (Pd.abs() @ av) + EPd @ av + u * f["out"].abs() + TINY
    if g is None:
        return b
    dP, delta = g["dP"].abs(), g["delta"].abs()
    BS = C * u * P * (dP + delta[..., None] + (P * dP).sum(-1, keepdim=True)) + EP * (dP + delta[..., None])
    b["dS"] = BS + u * g["dS"].abs() + TINY
    b["dQ_k"] = sc * (BS @ ak) + u * g["dQ_k"].abs() + TINY
    b["dQ"] = b["dQ_k"]
    b["dK"] = sc * (BS.transpose(-1, -2) @ aq) + u * g["dK"].abs() + TINY
    b["dV"] = (C * u * Pd.abs() + EPd).transpose(-1, -2) @ g["dO"].abs() + u * g["dV"].abs() + TINY
    if f["pe"] is not None:
        BQP = scatter_qp(BS, f["maxpos"])
        b["dQP"] = BQP + u * g["dQP"].abs() + TINY
        b["dQ"] = b["dQ_k"] + sc * (BQP @ f["pe"].abs()) + u * g["dQ"].abs()
        b["dPE"] = sc * torch.einsum("bhir,bhic->rc", BQP, aq) + u * g["dPE"].abs() + TINY
    return b


# ============================================================================================ decode (Tq = 1)
DCH = 64  # keys per split of st5_attn_decode_fwd


def decode_forward(q, k, v, *, scale, key_pad=None):
    """st5_attn_decode_fwd: q [B, H, 64], k / v [B, H, Tk, 64] -> out [B, H, 64] and P [B, H, Tk] = softmax over the
    unmasked keys of each (b, h). A (b, h) with every key masked gives zeros (out and P), as the header states."""
    f = forward(q[:, :, None], k, v, scale=scale, key_pad=key_pad)
    dead = ~f["ok"].any(-1)                                    # [B, H, 1]
    f["P"] = f["P"].masked_fill(dead[..., None], 0.0)
    f["Pd"] = f["P"]
    f["out"] = f["out"].masked_fill(dead[..., None], 0.0)
    f["dead"] = dead[..., 0]
    return f


def decode_bounds(f, *, u):
    """Elementwise bounds of out (storage unit u) and the fp32 probabilities, from `score_error` (64-term dot
    products: <= 8 sequential products per lane + 4 shuffle levels; the exponent; the merge factor exp(m_s - M)) and the
    fp32 sums: within a split, the denominator is a 5-level shuffle tree plus 4 warp partials and each output channel
    <= 8 sequential keys per lane, <= 2 shuffle levels and 4 warp partials; the splits are then merged in index order,
    one more level each (depth ns)."""
    P, av = f["P"], f["v"].abs()
    ns = -(-f["k"].shape[2] // DCH)
    es = score_error(f, 64.0)
    el = es.amax(-1, keepdim=True) + (ns + 16) * 2.0 ** -24          # relative error of the denominator L
    EP = P * (es + el + 2 * 2.0 ** -24)
    b = {"P": (EP + TINY)[:, :, 0]}
    b["out"] = ((ns + 24) * 2.0 ** -24 * (P @ av) + EP @ av + u * f["out"].abs() + TINY)[:, :, 0]
    return b


def check(name, got, ref, bound, dims="bhij", report=None):
    """Assert |got - ref| <= bound elementwise (NaN / inf in got fails). Names the first failing index and the largest
    err / bound; returns that ratio (and records it in `report[name]`)."""
    got = got.to(F64)
    ref = ref.to(F64)
    err = (got - ref).abs()
    ratio = err / bound
    ratio = torch.where(torch.isfinite(got), ratio, torch.full_like(ratio, math.inf))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    if report is not None:
        report[name] = max(report.get(name, 0.0), worst)
    if not worst <= 1.0:
        bad = torch.nonzero(~(ratio <= 1.0))
        first = tuple(int(t) for t in bad[0])
        where = ", ".join(f"{c}={t}" for c, t in zip(dims, first))
        raise AssertionError(f"{name}: {bad.shape[0]} of {ratio.numel()} elements out of bound; first ({where}): "
                             f"got {float(got[first]):.6g} ref {float(ref[first]):.6g} bound "
                             f"{float(bound[first]):.3g}; max err/bound {worst:.3g}")
    return worst


def make_inputs(B, H, Tq, Tk, *, std=3.0, seed=0, maxpos=0, probe=False, dtype=torch.bfloat16):
    """q, k, v [B, H, T, 64] and the position table [2 maxpos, 64] (fp32 master copy), rounded to `dtype`, so that the
    score has standard deviation about `std` (scale = 1/8). probe: k = 0 and only the table carries the score."""
    gen = torch.Generator().manual_seed(seed)
    sig = math.sqrt(std)  # scale * q.k over 64 channels: std = sig^2
    q = (torch.randn(B, H, Tq, 64, generator=gen) * sig).to(dtype)
    k = (torch.randn(B, H, Tk, 64, generator=gen) * sig).to(dtype)
    v = torch.randn(B, H, Tk, 64, generator=gen).to(dtype)
    pe = None
    if maxpos:
        pe = torch.randn(2 * maxpos, 64, generator=gen) * (sig if probe else sig * 0.5)
        if probe:
            k = torch.zeros_like(k)
    return q, k, v, pe
