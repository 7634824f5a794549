"""fp64 statement of st5_beam_topk's candidate scores with elementwise bounds, and a rank checker for one sentence's
candidate list (include/speecht5_b200.h). CPU only; no import of speecht5_b200.

The score of flat candidate f = beam * V + v of sentence s (row r = s K + beam) is
    z = x_v it - logsumexp_w(x_w it) (+ mask_v) (+ cum_r for t > 0)
in float64 on the exact inputs (bf16 logits widen exactly; `it` is the fp32 value of inv_temp), with eos -> -inf while
t < min_len, a row holding NaN or +inf -> every entry -inf (as log_softmax does), every v != eos -> -inf once
t >= max_len. A score that is -inf here is -inf on the device, exactly.

beam_row_topk computes in fp32, per row (a_v = x_v it, d_v = a_v - m, m = max_w a_w, p = softmax(a), u = 2^-24):
    y_v = fl(x_v it)                      |err| <= u |a_v|      (with FMA contraction y is never rounded: covered)
    d_v = fl(y_v - m)                     |err| <= u |d_v|
    e_v = expf(d_v)                       2 ulp (CUDA, no fast math): relative 4u, plus u |d_v| carried from d_v
    l   = sum e_v                         ceil(V / 256) sequential terms per thread, 5 shuffle levels, 8 warp partials
                                          added to 0 in order: relative (ceil(V / 256) + 12) u
    lse = logf(l)                         1 ulp: 2u |lse|; and d(log l) = relative error of l
    lp  = fl(d_v - lse), + mask, + cum    one rounding each: u |lp|, u |lp + mask|, u |z|
so, to first order,
    |score - z| <= u (|a_v| + |d_v| + sum_w p_w (|a_w| + |d_w|) + 4 + ceil(V / 256) + 12 + 2 |lse|
                      + |lp_v| + |lp_v + mask_v| + [t > 0] |z_v|) * (1 + 2^-10)
(the factor covers the second-order products; lse = log sum exp(d)). The error of logsumexp reaches every entry of the
row; the rest is the entry's own. At V = 81 and |z| ~ 10 this is about 2e-6; at V = 32768, 1e-5.

`check_sentence` asserts what the kernel's exact selection implies for one sentence's device lists (score, token,
beam)[:n], given z and the bound b of every flat candidate:
  - the flats are distinct and in range; a device score is -inf exactly when z is, never NaN, else |score - z| <= b;
  - the device scores do not increase; for picks i < j, z_j <= z_i + b_i + b_j (the order is exact wherever the fp64 gap
    exceeds the two bounds);
  - the i-th pick's z is within b_i + bmax of the fp64 i-th best, bmax the largest bound near the cut;
  - a candidate not picked has z <= z_last + b + b_last;
  - candidates whose inputs are bit-identical (`same`: same x, mask and eos status in rows with identical logits and
    cum; every -inf) come out in ascending flat index, picked ones before those left out."""
import math

import numpy as np
import torch

F64 = torch.float64
U = 2.0 ** -24
SECOND_ORDER = 1.0 + 2.0 ** -10


def scores(x, cum, mask, inv_temp, eos, t, min_len, max_len, K):
    """fp64 z [B, F] (F = V at t == 0: beam 0 only, else K V) and the elementwise bound [B, F] (0 where z = -inf)."""
    BK, V = x.shape
    B = BK // K
    it = float(np.float32(inv_temp))
    xd = x.to(F64)
    a = xd * it
    bad = torch.isnan(a).any(1) | (a == math.inf).any(1)
    a = torch.where(bad[:, None], torch.zeros_like(a), a)
    m = a.amax(1, keepdim=True)
    dead = bad | (m[:, 0] == -math.inf)
    m = torch.where(dead[:, None], torch.zeros_like(m), m)
    d = a - m
    lse = torch.log(torch.exp(d).sum(1, keepdim=True))
    lp = d - lse
    p = torch.exp(lp)
    fin = torch.isfinite(a)
    aa, ad = torch.where(fin, a.abs(), 0.0), torch.where(fin, d.abs(), 0.0)
    row_err = (p * (aa + ad)).sum(1, keepdim=True) + 4 + math.ceil(V / 256) + 12 + 2 * lse.abs()
    lp = torch.where(dead[:, None], torch.full_like(lp, -math.inf), lp)
    if t < min_len:
        lp[:, eos] = -math.inf
    lpm = lp + mask.to(F64)[None]
    if t >= max_len:
        keep = lpm[:, eos].clone()
        lpm.fill_(-math.inf)
        lpm[:, eos] = keep
    z = lpm + (cum.to(F64)[:, None] if t > 0 else 0.0)
    err = aa + ad + row_err + lp.abs() + lpm.abs() + (z.abs() if t > 0 else 0.0)
    bnd = torch.where(torch.isfinite(z), err * U * SECOND_ORDER, torch.zeros_like(z))
    if t == 0:
        return z.view(B, K, V)[:, 0], bnd.view(B, K, V)[:, 0]
    return z.reshape(B, K * V), bnd.reshape(B, K * V)


def emulate(x, cum, mask, inv_temp, eos, t, min_len, max_len, fma=False):
    """The kernel's row scores [BK, V] in fp32 (numpy), in its order of operations: strided per-thread sums over 256
    threads, the xor shuffle tree, the 8 warp partials in order. fma: y - m with one rounding."""
    f32 = np.float32
    xs = x.float().numpy().astype(f32)
    BK, V = xs.shape
    it = f32(inv_temp)
    with np.errstate(all="ignore"):
        y = (xs * it).astype(f32)
        m = y.max(1, keepdims=True)
        if fma:
            d = (xs.astype(np.float64) * float(it) - m.astype(np.float64)).astype(f32)
        else:
            d = (y - m).astype(f32)
        e = np.exp(d).astype(f32)
        nt = -(-V // 256)
        pad = np.zeros((BK, nt * 256), f32)
        pad[:, :V] = e
        acc = np.zeros((BK, 256), f32)
        for i in range(nt):
            acc = (acc + pad[:, i * 256:(i + 1) * 256]).astype(f32)
        w = acc.reshape(BK, 8, 32)
        lane = np.arange(32)
        for o in (16, 8, 4, 2, 1):
            w = (w + w[:, :, lane ^ o]).astype(f32)
        l = np.zeros(BK, f32)
        for i in range(8):
            l = (l + w[:, i, 0]).astype(f32)
        lse = np.log(l).astype(f32)[:, None]
        lp = (d - lse).astype(f32)
    if t < min_len:
        lp[:, eos] = -np.inf
    lp[np.isnan(lp)] = -np.inf
    lp = (lp + mask.numpy().astype(f32)[None]).astype(f32)
    if t >= max_len:
        keep = lp[:, eos].copy()
        lp[:] = -np.inf
        lp[:, eos] = keep
    if t > 0:
        lp = (lp + cum.numpy().astype(f32)[:, None]).astype(f32)
    return torch.from_numpy(lp)


def same_inputs(x, cum, mask, eos, K, s, t):
    """same(f, c) for sentence s: flat candidates whose device scores are bit-identical by construction -- equal logit
    and mask bits and eos status, in rows whose logits (all V) and cum are bit-identical."""
    V = x.shape[1]
    w = torch.int16 if x.dtype == torch.bfloat16 else torch.int32
    rows = x[s * K:(s + 1) * K].contiguous().view(w).to(torch.int64)
    cb = cum[s * K:(s + 1) * K].contiguous().view(torch.int32).to(torch.int64)
    if t == 0:
        cb = torch.zeros_like(cb)
    _, grp = torch.unique(torch.cat([rows, cb[:, None]], 1), dim=0, return_inverse=True)
    mb = mask.contiguous().view(torch.int32).to(torch.int64)

    def same(f, c):
        b0, v0 = divmod(int(f), V)
        bc, vc = c // V, c % V
        return (grp[bc] == grp[b0]) & (rows[bc, vc] == rows[b0, v0]) & (mb[vc] == mb[v0]) & ((vc == eos) == (v0 == eos))
    return same


def check_sentence(z, bnd, score, token, beam, V, same=None, what=""):
    """Assert that the device list (score, token, beam)[:n] is the kernel's exact top n of the flat candidates with fp64
    scores z [F] and bounds bnd [F] (see the module docstring). Returns the largest |score - z| / bound."""
    z, bnd = z.to(F64), bnd.to(F64)
    F = z.numel()
    s = torch.as_tensor(score).to(F64)
    n = s.numel()
    f = torch.as_tensor(beam).long() * V + torch.as_tensor(token).long()
    assert bool(((torch.as_tensor(token) >= 0) & (torch.as_tensor(token) < V)).all()), f"{what}: token out of range"
    assert bool(((f >= 0) & (f < F)).all()), f"{what}: candidate out of range {f.tolist()}"
    assert len(set(f.tolist())) == n, f"{what}: a (beam, token) pair picked twice {f.tolist()}"
    assert not bool(torch.isnan(s).any()), f"{what}: NaN score"
    zi, bi = z[f], bnd[f]
    ninf = zi == -math.inf
    assert torch.equal(s == -math.inf, ninf), f"{what}: -inf where the fp64 score is not (or the reverse)"
    err = (s - zi).abs()[~ninf]
    worst = float((err / bi[~ninf]).max()) if bool((~ninf).any()) else 0.0
    assert worst <= 1.0, f"{what}: a score off its own pair's fp64 score by {worst:.3g} x bound"
    assert bool((s[:-1] >= s[1:]).all()), f"{what}: device scores not descending"
    # pairwise order: i < j -> z_j <= z_i + b_i + b_j
    zz = torch.where(ninf, torch.full_like(zi, -1e300), zi)
    late = zz[None, :] > zz[:, None] + bi[:, None] + bi[None, :]
    late = torch.triu(late, 1)
    if bool(late.any()):
        i, j = (int(q) for q in torch.nonzero(late)[0])
        raise AssertionError(f"{what}: pick {j} (fp64 {float(zi[j]):.9g}) ranked after pick {i} "
                             f"(fp64 {float(zi[i]):.9g}) beyond the bounds")
    # rank: the i-th pick against the fp64 i-th best
    zs = torch.sort(z, descending=True).values[:n]
    fin = torch.isfinite(z)
    near = fin & (z >= zs[-1] - 2 * float(bnd.max())) if bool(torch.isfinite(zs[-1])) else fin
    bmax = float(bnd[near].max()) if bool(near.any()) else 0.0
    assert torch.equal(zs == -math.inf, ninf), f"{what}: a -inf pick while a finite candidate is left, or the reverse"
    off = (zi - zs).abs()[~ninf] > (bi + bmax)[~ninf]
    assert not bool(off.any()), f"{what}: pick {int(torch.nonzero(off)[0])} is not within bound of that rank's best"
    # the cut: nothing left out beats the last pick beyond the bounds
    out = torch.ones(F, dtype=torch.bool)
    out[f] = False
    if bool(ninf[-1]):
        assert not bool(fin[out].any()), f"{what}: a finite candidate left out behind a -inf pick"
    else:
        beat = out & fin & (z > zi[-1] + bnd + bi[-1])
        if bool(beat.any()):
            c = int(torch.nonzero(beat)[0])
            raise AssertionError(f"{what}: candidate {c} (fp64 {float(z[c]):.9g}) left out, better than the last pick "
                                 f"(fp64 {float(zi[-1]):.9g}) beyond the bounds")
    # bit-identical inputs: ascending flat index, picked before left out
    idx = torch.arange(F)
    for i in range(n):
        if bool(ninf[i]):
            eq = z == -math.inf
        else:
            eq = z == zi[i]
            if same is not None:
                c = idx[eq]
                keep = same(int(f[i]), c)
                eq = torch.zeros(F, dtype=torch.bool)
                eq[c[keep]] = True
        eq[f[i]] = False
        lower = eq & (idx < f[i])
        if bool((lower & out).any()):
            raise AssertionError(f"{what}: tie broken the wrong way: candidate {int(torch.nonzero(lower & out)[0])} "
                                 f"left out while the identical, higher flat {int(f[i])} was picked")
        pos = {int(q): k for k, q in enumerate(f.tolist())}
        for c in torch.nonzero(eq & ~out).flatten().tolist():
            if (c < int(f[i])) != (pos[c] < i):
                raise AssertionError(f"{what}: tie between flats {int(f[i])} and {c} in the wrong order")
    return worst
