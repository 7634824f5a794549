"""CPU: tests/attention_ref.py (the fp64 statement the attention kernels are checked against) is itself checked here.

1. Against an independent statement: pos_k materialised as [Tq, Tk, 64] (multihead_attention.py:346-353), the
   softmax / dropout / PV written out plainly, and every gradient taken by torch autograd.
2. Bound sensitivity: at shapes and seeds of tests/test_attention_contract_gpu.py, each of a list of one-line kernel
   defects, applied to the fp64 statement, leaves the bf16 bound somewhere. So a kernel with that defect cannot pass."""
import math

import pytest
import torch

import attention_ref as R
import dropout_ref as D

F64 = torch.float64


def _independent(q, k, v, pe, maxpos, scale, causal, key_pad, keep, dscale, dO, dP_ext):
    q, k, v = (t.to(F64).clone().requires_grad_() for t in (q, k, v))
    pe = pe.to(F64).clone().requires_grad_() if pe is not None else None
    B, H, Tq, _ = q.shape
    Tk = k.shape[2]
    outs, probs = [], []
    for b in range(B):
        ob, pb = [], []
        for h in range(H):
            qi, kj = q[b, h], k[b, h]
            sc = qi @ kj.T
            if pe is not None:
                idx = torch.tensor([[min(max(i - j, -maxpos), maxpos - 1) + maxpos for j in range(Tk)]
                                    for i in range(Tq)])
                pos_k = pe[idx]  # [Tq, Tk, 64]
                sc = sc + torch.einsum("ic,ijc->ij", qi, pos_k)
            sc = sc * scale
            for i in range(Tq):
                for j in range(Tk):
                    if (causal and j > i) or (key_pad is not None and key_pad[b, j]):
                        sc = sc.index_put((torch.tensor(i), torch.tensor(j)), torch.tensor(-math.inf, dtype=F64))
            p = torch.softmax(sc, -1)
            ob.append((p * keep[b, h] * dscale) @ v[b, h])
            pb.append(p)
        outs.append(torch.stack(ob))
        probs.append(torch.stack(pb))
    out, P = torch.stack(outs), torch.stack(probs)
    loss = (out * dO).sum() + (0 if dP_ext is None else (P * dP_ext).sum())
    loss.backward()
    return out.detach(), P.detach(), q.grad, k.grad, v.grad, (pe.grad if pe is not None else None)


@pytest.mark.parametrize("case", [
    dict(B=2, H=2, Tq=9, Tk=9, maxpos=3, causal=False, pad=True, drop=0.0, ext=True),
    dict(B=1, H=2, Tq=11, Tk=11, maxpos=4, causal=False, pad=False, drop=0.3, ext=False),
    dict(B=2, H=1, Tq=7, Tk=7, maxpos=0, causal=True, pad=True, drop=0.2, ext=True),
    dict(B=1, H=2, Tq=5, Tk=12, maxpos=0, causal=False, pad=True, drop=0.0, ext=True),
])
def test_reference_matches_autograd_statement(case):
    B, H, Tq, Tk, maxpos = case["B"], case["H"], case["Tq"], case["Tk"], case["maxpos"]
    gen = torch.Generator().manual_seed(3)
    q, k, v = (torch.randn(B, H, t, 64, generator=gen, dtype=F64) * 0.3 for t in (Tq, Tk, Tk))
    pe = torch.randn(2 * maxpos, 64, generator=gen, dtype=F64) * 0.3 if maxpos else None
    key_pad = None
    if case["pad"]:
        key_pad = torch.zeros(B, Tk, dtype=torch.bool)
        key_pad[-1, Tk - 3:] = True
    keep = R.keep_mask(B, H, Tq, Tk, case["drop"], 11, 5)
    dO = torch.randn(B, H, Tq, 64, generator=gen, dtype=F64)
    dP_ext = torch.randn(B, H, Tq, Tk, generator=gen, dtype=F64) if case["ext"] else None
    f = R.forward(q, k, v, scale=0.125, pe=pe, maxpos=maxpos, causal=case["causal"], key_pad=key_pad,
                  drop_p=case["drop"], seed=11, offset=5)
    g = R.backward(f, dO, dP_ext)
    out, P, dq, dk, dv, dpe = _independent(q, k, v, pe, maxpos, 0.125, case["causal"], key_pad, keep,
                                           D.drop_scale(case["drop"]), dO, dP_ext)
    for name, a, b in (("out", f["out"], out), ("P", f["P"], P), ("dQ", g["dQ"], dq), ("dK", g["dK"], dk),
                       ("dV", g["dV"], dv)) + ((("dPE", g["dPE"], dpe),) if maxpos else ()):
        assert torch.allclose(a, b, rtol=1e-10, atol=1e-12), name
    # side outputs of the fused kernels: psave = exp(s - max) with P = e * inv_l, lse = log sum exp(s)
    assert torch.allclose(f["e"] * f["inv_l"][..., None], P, rtol=1e-12, atol=1e-14)
    s = f["s"]
    assert torch.allclose(f["lse"], torch.logsumexp(s, -1), rtol=1e-12)
    # delta = dO . out + sum P dP_ext; the head-major scatter is a permutation of the (b, h, i) one
    d2 = (dO * f["out"]).sum(-1) + (0 if dP_ext is None else (P * dP_ext).sum(-1))
    assert torch.allclose(g["delta"], d2, rtol=1e-10, atol=1e-12)
    if maxpos:
        hm = R.head_major(g["dQP"])
        assert torch.equal(hm[1, 0], g["dQP"][0, 1])


# --------------------------------------------------------------------------------------------- bound sensitivity
def _case(B, H, T, *, Tk=None, causal=False, maxpos=0, probe=False, pad=False, drop=0.0, seed=0):
    Tk = Tk or T
    q, k, v, pe = R.make_inputs(B, H, T, Tk, seed=seed, maxpos=maxpos, probe=probe)
    if pe is not None:
        pe = pe.to(torch.bfloat16)
    key_pad = None
    if pad:
        key_pad = torch.zeros(B, Tk, dtype=torch.bool)
        key_pad[-1, max(1, Tk // 2):] = True
    kw = dict(scale=0.125, pe=pe, maxpos=maxpos, causal=causal, key_pad=key_pad, drop_p=drop, seed=77, offset=3)
    f = R.forward(q, k, v, **kw)
    gen = torch.Generator().manual_seed(seed + 1)
    dO = torch.randn(B, H, T, 64, generator=gen).to(torch.bfloat16)
    return (q, k, v), kw, f, dO


def _exceeds(got, ref, bound):
    return bool(((got - ref).abs() > bound).any())


@pytest.mark.parametrize("j", ["63", "64", "last"])
def test_one_dropped_key_exceeds_out_bound(j):
    (q, k, v), kw, f, dO = _case(2, 2, 130)
    b = R.bounds(f, u=R.U_BF16, C=R.C_BF16)
    jj = {"63": 63, "64": 64, "last": 129}[j]
    pad = torch.zeros(2, 130, dtype=torch.bool)
    pad[:, jj] = True
    m = R.forward(q, k, v, **dict(kw, key_pad=pad))
    assert _exceeds(m["out"], f["out"], b["out"])


def test_shifted_causal_diagonal_exceeds_out_bound():
    (q, k, v), kw, f, dO = _case(2, 2, 130, causal=True)
    b = R.bounds(f, u=R.U_BF16, C=R.C_BF16)
    # j < i instead of j <= i (rows keep at least one key)
    pad = None
    m = R.forward(q[:, :, 1:], k[:, :, :-1], v[:, :, :-1], **dict(kw, key_pad=pad))
    assert _exceeds(m["out"], f["out"][:, :, 1:], b["out"][:, :, 1:])


@pytest.mark.parametrize("T,maxpos", [(199, 64), (65, 8), (781, 160)])
def test_rpe_clamp_off_by_one_exceeds_out_bound(T, maxpos, monkeypatch):
    (q, k, v), kw, f, dO = _case(1, 2, T, maxpos=maxpos, probe=True)
    b = R.bounds(f, u=R.U_BF16, C=R.C_BF16)
    orig = R.rel_index

    def clamp_low(Tq, Tk, mp, rows=None):  # clamp(i - j, -maxpos + 1, maxpos - 1): the lowest table row is never used
        return orig(Tq, Tk, mp, rows).clamp(min=1)
    monkeypatch.setattr(R, "rel_index", clamp_low)
    m = R.forward(q, k, v, **kw)
    assert _exceeds(m["out"], f["out"], b["out"])

    def clamp_high(Tq, Tk, mp, rows=None):  # clamp at maxpos - 2
        return orig(Tq, Tk, mp, rows).clamp(max=2 * mp - 2)
    monkeypatch.setattr(R, "rel_index", clamp_high)
    m = R.forward(q, k, v, **kw)
    assert _exceeds(m["out"], f["out"], b["out"])


def test_rpe_index_off_by_one_across_key_window_exceeds_out_bound(monkeypatch):
    (q, k, v), kw, f, dO = _case(1, 2, 199, maxpos=64, probe=True)
    b = R.bounds(f, u=R.U_BF16, C=R.C_BF16)
    orig = R.rel_index

    def shifted(Tq, Tk, mp, rows=None):  # keys of the second 64-key block read the neighbouring table row
        idx = orig(Tq, Tk, mp, rows).clone()
        idx[:, 64:128] = (idx[:, 64:128] + 1).clamp(max=2 * mp - 1)
        return idx
    monkeypatch.setattr(R, "rel_index", shifted)
    m = R.forward(q, k, v, **kw)
    assert _exceeds(m["out"], f["out"], b["out"])


def test_zeroed_last_query_tile_exceeds_out_bound():
    (q, k, v), kw, f, dO = _case(2, 2, 130)
    b = R.bounds(f, u=R.U_BF16, C=R.C_BF16)
    got = f["out"].clone()
    got[:, :, 128:] = 0
    assert _exceeds(got, f["out"], b["out"])


def test_delta_without_external_dp_exceeds_gradient_bounds():
    (q, k, v), kw, f, dO = _case(2, 2, 130)
    gen = torch.Generator().manual_seed(9)
    ext = torch.randn(2, 2, 130, 130, generator=gen)
    g = R.backward(f, dO, ext)
    b = R.bounds(f, g, u=R.U_BF16, C=R.C_BF16)
    P, dP = f["P"], g["dP"]
    dS_bad = P * (dP - (P * (dP - ext.to(F64))).sum(-1, keepdim=True))
    assert _exceeds(dS_bad, g["dS"], b["dS"])
    assert _exceeds(0.125 * dS_bad @ f["k"], g["dQ"], b["dQ"])
    assert _exceeds(0.125 * dS_bad.transpose(-1, -2) @ f["q"], g["dK"], b["dK"])


def test_flipped_psave_sign_bit_exceeds_dv_bound():
    (q, k, v), kw, f, dO = _case(2, 2, 130, drop=0.2)
    g = R.backward(f, dO)
    b = R.bounds(f, g, u=R.U_BF16, C=R.C_BF16)
    # flip the dropout decision of the most probable element of one row
    i = 70
    j = int(f["P"][1, 1, i].argmax())
    keep = f["keep"].clone()
    keep[1, 1, i, j] = ~keep[1, 1, i, j]
    m = R.forward(q, k, v, **dict(kw, keep=keep))
    gm = R.backward(m, dO)
    assert _exceeds(gm["dV"], g["dV"], b["dV"])


def test_masked_key_gradient_exceeds_bound():
    (q, k, v), kw, f, dO = _case(2, 2, 130, pad=True)
    g = R.backward(f, dO)
    b = R.bounds(f, g, u=R.U_BF16, C=R.C_BF16)
    for name in ("dK", "dV"):
        got = g[name].clone()
        got[1, 0, 100] += 1e-6  # key 100 of utterance 1 is padded
        assert _exceeds(got, g[name], b[name]), name
