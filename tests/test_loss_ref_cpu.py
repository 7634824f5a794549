"""The fp64 statement of tests/loss_ref.py checked on its own (no GPU): against independent statements (torch's
ctc_loss on log_softmax, F.normalize and oracle/speaker_oracle.py in fp64 autograd, and the reference's own
Tacotron2Loss and GuidedMultiHeadAttentionLoss), and by showing that each of a list of one-line kernel defects, put into
the statement, leaves the bound the GPU test uses at that test's shapes."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

import loss_ref as R

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_loader as rl  # noqa: E402
from oracle import speaker_oracle as so  # noqa: E402

F64 = torch.float64
needs_ref = pytest.mark.skipif(not rl.available(), reason="reference tree not available")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _f32(t):
    return t.float().double()


# ============================================================================================ CTC
def ctc_case(T, B, V, tls, ils, blank, seed=0, scale=1.0, repeat=False):
    """logits [T, B, V] (fp32 values), targets avoiding `blank`; `repeat`: runs of equal labels."""
    g = _gen(seed)
    x = _f32(torch.randn(T, B, V, generator=g, dtype=F64) * scale)
    labels = [k for k in range(V) if k != blank]
    tg = []
    for b, L in enumerate(tls):
        idx = torch.randint(0, len(labels), (L,), generator=g)
        t = torch.tensor([labels[i] for i in idx], dtype=torch.long)
        if repeat and L >= 4:
            t[1] = t[0]
            t[3] = t[2]
        tg.append(t)
    return x, tg, list(ils)


def _torch_ctc(x, tg, ils, blank, zero_infinity):
    xa = x.clone().requires_grad_()
    lp = F.log_softmax(xa, -1)
    tl = torch.tensor([len(t) for t in tg])
    flat = torch.cat(tg) if sum(len(t) for t in tg) else torch.zeros(0, dtype=torch.long)
    nll = F.ctc_loss(lp, flat, torch.tensor(ils), tl, blank=blank, reduction="none", zero_infinity=zero_infinity)
    nll.sum().backward()
    return nll.detach(), xa.grad


@pytest.mark.parametrize("zero_infinity", [False, True])
@pytest.mark.parametrize("blank", ["first", "last", "middle"])
def test_ctc_matches_torch_ctc_loss(blank, zero_infinity):
    T, B, V = 23, 5, 11
    bl = {"first": 0, "last": V - 1, "middle": 5}[blank]
    x, tg, ils = ctc_case(T, B, V, [4, 0, 7, 10, 3], [23, 17, 20, 9, 1], bl, seed=1, repeat=True)
    # utterance 3: 10 labels with repeats in 9 frames (infeasible); utterance 4: 3 labels in one frame (infeasible)
    ref = R.ctc(x, tg, ils, blank=bl, zero_infinity=zero_infinity, S_max=21)
    nll, grad = _torch_ctc(x, tg, ils, bl, zero_infinity)
    fe = ref["feasible"]
    assert fe.tolist() == [True, True, True, False, False]
    assert torch.allclose(ref["nll"][fe], nll[fe], rtol=1e-12, atol=1e-12)
    assert torch.equal(ref["nll"][~fe], nll[~fe])  # +inf, or 0 under zero_infinity
    feas = [b for b in range(B) if fe[b]]
    assert torch.allclose(ref["grad"][:, feas], grad[:, feas], rtol=1e-10, atol=1e-12)
    if zero_infinity:  # torch zeroes the infeasible utterances' gradient too
        inf = [b for b in range(B) if not fe[b]]
        assert float(grad[:, inf].abs().max()) == 0.0 and float(ref["grad"][:, inf].abs().max()) == 0.0
    # the bound is a small fraction of the values it bounds
    assert float((ref["b_nll"][fe] / ref["nll"][fe].abs()).max()) < 1e-4
    assert float(ref["b_grad"].max()) < 1e-3


def test_ctc_s_max_and_lengths():
    T, B, V = 9, 4, 6
    x, tg, ils = ctc_case(T, B, V, [3, 4, 0, 2], [9, 30, 0, 5], 0, seed=2)
    ref = R.ctc(x, tg, ils, blank=0, zero_infinity=False, S_max=8)
    # S = 9 > S_max = 8: reported infeasible; input length 0: infeasible; 30 > T counts as T
    assert ref["feasible"].tolist() == [True, False, False, True]
    assert math.isinf(ref["nll"][1]) and math.isinf(ref["nll"][2])
    ref9 = R.ctc(x, tg, [9, 9, 0, 5], blank=0, zero_infinity=False, S_max=9)
    ref30 = R.ctc(x, tg, [9, 30, 0, 5], blank=0, zero_infinity=False, S_max=9)
    assert torch.equal(ref9["nll"], ref30["nll"]) and torch.equal(ref9["grad"], ref30["grad"])
    assert float(ref["grad"][5:, 3].abs().max()) == 0.0  # rows t >= input length


# ============================================================================================ TTS loss
def tts_case(B, L, D, olens, seed=3, Ly=None, lab_w=None, big_logits=False):
    g = _gen(seed)
    Ly = Ly or L
    a = _f32(torch.randn(B, L, D, generator=g, dtype=F64))
    bf = _f32(torch.randn(B, L, D, generator=g, dtype=F64))
    ys = _f32(torch.randn(B, Ly, D, generator=g, dtype=F64))
    x = _f32(torch.randn(B, L, generator=g, dtype=F64) * (30.0 if big_logits else 2.0))
    labels = (torch.rand(B, lab_w or L, generator=g, dtype=F64) < 0.2).to(F64)
    # exact zeros of after - ys (sign(0))
    a[0, 0, : D // 2] = ys[0, 0, : D // 2]
    return a, bf, x, ys, labels, torch.tensor(olens)


def _tacotron(a, bf, x, ys, labels, olens, r, pw):
    ns = rl.load()
    crit = ns.tts_loss.Tacotron2Loss(use_masking=True, use_weighted_masking=False, bce_pos_weight=pw).double()
    if r > 1:  # compute_loss (:162-168)
        olens = olens.new([o - o % r for o in olens])
        m = max(olens)
        ys, labels = ys[:, :m], labels[:, :m]
        labels = torch.scatter(labels, 1, (olens - 1).unsqueeze(1), 1.0)
    ts = [t.clone().requires_grad_() for t in (a, bf, x)]
    l1, l2, bce = crit(ts[0], ts[1], ts[2], ys, labels, olens)
    return (l1, l2, bce), ts


@needs_ref
@pytest.mark.parametrize("r,olens", [(1, [9, 4, 7]), (2, [9, 10, 3]), (3, [11, 12, 5])])
@pytest.mark.parametrize("pw", [1.0, 5.0])
def test_tts_matches_reference_tacotron2_loss(r, olens, pw):
    L = max(o - o % r for o in olens)
    a, bf, x, ys, labels, ol = tts_case(3, L, 7, olens, seed=r)
    (l1, l2, bce), ts = _tacotron(a, bf, x, ys, labels, ol, r, pw)
    g = (0.7, -1.3, 2.1)
    st = R.tts_loss(a, bf, x, ys, labels, ol, r=r, pos_weight=pw, g=g)
    ref = torch.stack([l1.detach(), l2.detach(), bce.detach()])
    assert torch.allclose(st["out"], ref, rtol=1e-12, atol=1e-14)
    (g[0] * l1 + g[1] * l2 + g[2] * bce).backward()
    assert torch.allclose(st["d_after"], ts[0].grad, rtol=1e-10, atol=1e-14)
    assert torch.allclose(st["d_before"], ts[1].grad, rtol=1e-10, atol=1e-14)
    assert torch.allclose(st["d_logits"], ts[2].grad, rtol=1e-10, atol=1e-14)


@needs_ref
@pytest.mark.parametrize("r,heads,nl", [(1, 2, 1), (2, 3, 2), (3, 4, 3)])
def test_guided_matches_reference_class(r, heads, nl):
    ns = rl.load()
    B, H = 3, 4
    olens = torch.tensor([21, 14, 9])
    ilens = torch.tensor([7, 13, 10])
    T_out, T_in = max(int(o) // r for o in olens), int(ilens.max())
    g = _gen(4)
    att = [_f32(torch.rand(B, H, T_out, T_in, generator=g, dtype=F64)) for _ in range(nl)]
    crit = ns.tts_loss.GuidedMultiHeadAttentionLoss(sigma=0.4, alpha=10.0)
    olens_in = olens.new([torch.div(o, r, rounding_mode="floor") for o in olens])
    ref = crit(torch.cat([a[:, :heads] for a in att], 1), ilens, olens_in)
    st = R.guided(att, ilens, olens, r=r, heads=heads, sigma=0.4, alpha=10.0)
    # the reference builds W in fp32 (torch.zeros default dtype)
    assert abs(st["out"] - float(ref)) <= 1e-6 * abs(float(ref))
    aa = [a.clone().requires_grad_() for a in att]
    crit2 = ns.tts_loss.GuidedMultiHeadAttentionLoss(sigma=0.4, alpha=10.0)
    crit2(torch.cat([a[:, :heads] for a in aa], 1), ilens, olens_in).backward()
    for a in aa:
        scale = float(st["datt"].abs().max())  # (fp32 W of the reference: absolute error ~ 1e-7 of the largest)
        assert torch.allclose(st["datt"], a.grad[:, :heads], rtol=1e-6, atol=1e-6 * scale)
        assert float(a.grad[:, heads:].abs().max()) == 0.0 if heads < H else True


# ============================================================================================ speaker head
@pytest.mark.parametrize("mode,easy", [(1, 0), (2, 0), (2, 1), (0, 0)])
def test_margin_ce_matches_speaker_oracle(mode, easy):
    B, N = 7, 13
    g = _gen(5)
    x = _f32(torch.rand(B, N, generator=g, dtype=F64) * 1.8 - 0.9)
    mt = torch.randint(0, N, (B,), generator=g)
    x[0, mt[0]] = -0.99  # below th = cos(pi - m)
    x[1, mt[1]] = -0.2   # between th and 0
    tgt = mt.clone()
    tgt[2] = 1  # ignore_index
    scale, m, eps = 30.0, 0.2, 0.1
    kind = {1: "amsoftmax", 2: "aamsoftmax"}.get(mode)
    xa = x.clone().requires_grad_()
    z = so.margin(xa, mt, kind, R.f32(m), R.f32(scale), bool(easy)) if mode else xa
    loss, nll, corr, tot = so.label_smoothed_ce(z, tgt, eps, ignore_index=1)
    f = R.margin_ce_fwd(x, mt if mode else None, tgt, mode=mode, scale=scale, margin=m, easy=easy, eps=eps,
                        ignore_index=1)
    assert torch.allclose(f["z"], z.detach(), rtol=1e-6, atol=1e-6)
    assert abs(float(f["loss"].sum()) - float(loss)) <= 1e-5 * abs(float(loss))
    assert abs(float(f["nll"].sum()) - float(nll)) <= 1e-5 * abs(float(nll))
    assert int(f["correct"].sum()) == corr and int(f["valid"].sum()) == tot
    ga, gn = 0.75, -0.5
    (ga * loss + gn * nll).backward()
    dx, edx = R.margin_ce_bwd(f, tgt, eps=eps, ignore_index=1, gstat=(ga, gn))
    assert torch.allclose(dx, xa.grad, rtol=1e-5, atol=1e-5)


def test_l2norm_matches_f_normalize():
    g = _gen(6)
    x = torch.randn(9, 33, generator=g, dtype=F64)
    x[4] = 1e-14  # clamped row
    xa = x.clone().requires_grad_()
    y = F.normalize(xa, p=2, dim=1)
    f = R.l2norm_fwd(x)
    assert torch.allclose(f["y"], y.detach(), rtol=1e-13, atol=0)
    dy = torch.randn(9, 33, generator=g, dtype=F64)
    y.backward(dy)
    dx, _ = R.l2norm_bwd(dy, f["y"], f["nrm"])
    assert torch.allclose(dx, xa.grad, rtol=1e-10, atol=1e-6)


def test_time_mean_matches_mean():
    x = torch.randn(3, 17, 37, generator=_gen(7), dtype=F64)
    y, _ = R.time_mean_fwd(x, R.U32)
    assert torch.allclose(y, x.mean(1), rtol=1e-14)
    xa = x.clone().requires_grad_()
    dy = torch.randn(3, 37, generator=_gen(8), dtype=F64)
    xa.mean(1).backward(dy)
    dx, _ = R.time_mean_bwd(dy, 17, R.U32)
    assert torch.allclose(dx, xa.grad, rtol=1e-14)


# ============================================================================================ defects leave the bound
# shapes below are cases of tests/test_loss_contract_gpu.py
def _ctc_gpu_case(repeat=False, blank=0):
    return ctc_case(40, 3, 33, [6, 9, 3], [40, 31, 25], blank, seed=11, repeat=repeat)


def test_ctc_skip_between_equal_labels_leaves_bound(monkeypatch):
    x, tg, ils = _ctc_gpu_case(repeat=True)
    ref = R.ctc(x, tg, ils, blank=0, zero_infinity=False, S_max=19)
    good_ext = R._ext

    def bad_ext(t, blank):
        lab, skip = good_ext(t, blank)
        skip[3::2] = True
        return lab, skip
    monkeypatch.setattr(R, "_ext", bad_ext)
    bad = R.ctc(x, tg, ils, blank=0, zero_infinity=False, S_max=19)
    assert R.exceeds(bad["nll"], ref["nll"], ref["b_nll"])


def test_ctc_beta_skip_on_wrong_neighbour_leaves_bound(monkeypatch):
    x, tg, ils = _ctc_gpu_case(repeat=True)
    ref = R.ctc(x, tg, ils, blank=0, zero_infinity=False, S_max=19)
    monkeypatch.setattr(R, "_beta_skip", lambda skip: skip)
    bad = R.ctc(x, tg, ils, blank=0, zero_infinity=False, S_max=19)
    assert R.exceeds(bad["grad"], ref["grad"], ref["b_grad"])


def test_ctc_row_and_length_defects_leave_bound():
    x, tg, ils = _ctc_gpu_case()
    ref = R.ctc(x, tg, ils, blank=0, zero_infinity=False, S_max=19)
    # rows t >= Tn not zeroed (softmax left there)
    bad = ref["grad"].clone()
    sm = torch.softmax(x, -1)
    bad[31:, 1] = sm[31:, 1]
    assert R.exceeds(bad, ref["grad"], ref["b_grad"])
    # Tn taken as T
    bad = R.ctc(x, tg, [40, 40, 40], blank=0, zero_infinity=False, S_max=19)
    assert R.exceeds(bad["nll"], ref["nll"], ref["b_nll"])


def test_ctc_blank_defects_leave_bound():
    V = 33
    x, tg, ils = _ctc_gpu_case(blank=V - 1)
    ref = R.ctc(x, tg, ils, blank=V - 1, zero_infinity=False, S_max=19)
    # blank hard-wired to 0 (the targets avoid V - 1 only)
    tg0 = [torch.where(t == 0, torch.ones_like(t), t) for t in tg]
    x0, _, _ = _ctc_gpu_case(blank=V - 1)
    ref0 = R.ctc(x0, tg0, ils, blank=V - 1, zero_infinity=False, S_max=19)
    bad0 = R.ctc(x0, tg0, ils, blank=0, zero_infinity=False, S_max=19)
    assert R.exceeds(bad0["nll"], ref0["nll"], ref0["b_nll"])
    # blank mass added to class 0
    pb = torch.softmax(x, -1)[..., V - 1] - ref["grad"][..., V - 1]
    pb = torch.where(ref["grad"].abs().sum(-1) > 0, pb, torch.zeros_like(pb))
    bad = ref["grad"].clone()
    bad[..., V - 1] += pb
    bad[..., 0] -= pb
    assert R.exceeds(bad, ref["grad"], ref["b_grad"])


def test_ctc_zero_infinity_on_raw_nll_leaves_bound():
    # an infeasible utterance (repeats, too few frames) under zero_infinity: its gradient must stay zero
    x, tg, ils = ctc_case(40, 3, 33, [6, 12, 3], [40, 13, 25], 0, seed=12, repeat=True)
    ref = R.ctc(x, tg, ils, blank=0, zero_infinity=True, S_max=25)
    assert ref["feasible"].tolist() == [True, False, True]
    bad = ref["grad"].clone()
    bad[:13, 1] = torch.softmax(x[:13, 1], -1)
    assert R.exceeds(bad, ref["grad"], ref["b_grad"])


def _tts_gpu_case(r=2):
    olens = [37, 40, 6, 41]  # olens % r != 0, olens < ... ; L = 41
    return tts_case(4, 41, 80, olens, seed=21), r


def test_tts_mask_and_label_defects_leave_bound(monkeypatch):
    (a, bf, x, ys, labels, ol), r = _tts_gpu_case()
    ref = R.tts_loss(a, bf, x, ys, labels, ol, r=r, pos_weight=5.0)
    # the mask on olens instead of olens - olens % r
    monkeypatch.setattr(R, "tts_valid", lambda olens, L, r_: (torch.arange(L)[None, :] < torch.as_tensor(olens)[:, None],
                                                              torch.as_tensor(olens) - torch.as_tensor(olens) % r_))
    bad = R.tts_loss(a, bf, x, ys, labels, ol, r=r, pos_weight=5.0)
    assert R.exceeds(bad["out"], ref["out"], ref["b_out"])
    monkeypatch.undo()
    # the forced label at ol instead of ol - 1
    good_st = R._stop_target

    def bad_st(lab, oln, r_):
        t = lab.clone()
        for b in range(t.shape[0]):
            if oln[b] < t.shape[1]:
                t[b, oln[b]] = 1.0
        return t
    monkeypatch.setattr(R, "_stop_target", bad_st)
    bad = R.tts_loss(a, bf, x, ys, labels, ol, r=r, pos_weight=5.0)
    assert R.exceeds(bad["out"], ref["out"], ref["b_out"])
    monkeypatch.setattr(R, "_stop_target", good_st)
    # pos_weight on the negative term
    monkeypatch.setattr(R, "_bce_terms", lambda x_, t, pw: t * R._softplus(-x_) + pw * (1 - t) * R._softplus(x_))
    bad = R.tts_loss(a, bf, x, ys, labels, ol, r=r, pos_weight=5.0)
    assert R.exceeds(bad["out"], ref["out"], ref["b_out"])


def test_tts_scale_and_sign_defects_leave_bound():
    (a, bf, x, ys, labels, ol), r = _tts_gpu_case()
    ref = R.tts_loss(a, bf, x, ys, labels, ol, r=r, pos_weight=5.0, g=(1.0, 0.5, 2.0))
    # /D missing from l1
    bad = ref["out"].clone()
    bad[0] *= 80
    assert R.exceeds(bad, ref["out"], ref["b_out"])
    # sign(0) = +1 in the L1 gradient (after == ys at [0, 0, :40])
    d = (a - ys[:, :41]) * ref["valid"][..., None]
    k1 = 1.0 / (ref["n"] * 80)
    bad = ref["d_after"] + torch.where((d == 0) & ref["valid"][..., None], torch.full_like(d, k1), torch.zeros_like(d))
    assert R.exceeds(bad, ref["d_after"], ref["b_d_after"])


def _guided_gpu_case():
    B, H, T_out, T_in, nl = 3, 4, 30, 17, 2
    g = _gen(31)
    att = [_f32(torch.rand(B, H, T_out, T_in, generator=g, dtype=F64)) for _ in range(nl)]
    return att, torch.tensor([17, 9, 12]), torch.tensor([60, 41, 25])


def test_guided_defects_leave_bound(monkeypatch):
    att, il, ol = _guided_gpu_case()
    ref = R.guided(att, il, ol, r=2, heads=3, sigma=0.4, alpha=10.0, g=1.5)
    # normaliser without heads * n_layers
    assert R.exceeds(torch.tensor(ref["out"] * 3 * 2), torch.tensor(ref["out"]), torch.tensor(ref["b_out"]))
    # datt non-zero in the columns [il, p_ld)
    W, _, _ = R.guided_w(9, 20, 20, 30, 17, 0.4)
    bad = ref["datt"].clone()
    bad[1, :, :20, 9:] = (1.5 * R.f32(10.0) / ref["gsum1"]) * W[:20, 9:]
    assert R.exceeds(bad, ref["datt"], ref["b_datt"])
    # W dividing by olens instead of olens / r
    monkeypatch.setattr(R, "_ol_w", lambda olen, r: int(olen))
    bad = R.guided(att, il, ol, r=2, heads=3, sigma=0.4, alpha=10.0, g=1.5)
    assert R.exceeds(torch.tensor(bad["out"]), torch.tensor(ref["out"]), torch.tensor(ref["b_out"]))


def _spk_gpu_case(N=257, B=6):
    g = _gen(41)
    x = _f32(torch.rand(B, N, generator=g, dtype=F64) * 1.6 - 0.8)
    mt = torch.randint(0, N, (B,), generator=g)
    return x, mt


def test_speaker_eps_and_tie_defects_leave_bound():
    x, mt = _spk_gpu_case()
    f = R.margin_ce_fwd(x, mt, mt, mode=2, scale=30.0, margin=0.2, easy=0, eps=0.1, ignore_index=-100)
    N = x.shape[1]
    # eps_i = eps / N instead of eps / (N - 1)
    eps_f = R.f32(0.1)
    bad_i = eps_f / N
    smooth = N * f["lse"] - f["z"].sum(1)
    bad = (1 - eps_f - bad_i) * f["nll"] + bad_i * smooth
    assert R.exceeds(bad, f["loss"], f["b_loss"])
    # an exact tie at the maximum: the lowest index wins
    xt = x.clone()
    xt[0, 5] = xt[0, 200] = 0.95
    f = R.margin_ce_fwd(xt, None, torch.full((6,), 5), mode=0, scale=1.0, margin=0.0, easy=0, eps=0.0,
                        ignore_index=-100)
    assert f["correct"][0] == 1.0
    rev = torch.argmax(xt.flip(1), 1)
    assert (N - 1 - int(rev[0])) == 200  # the highest index would score the row as wrong


def test_aam_threshold_with_ge_leaves_bound():
    x, mt = _spk_gpu_case()
    c = R.margin_consts(2, 30.0, 0.2)
    x[0, mt[0]] = c["th"]  # exactly at th: kept only with >=
    f = R.margin_ce_fwd(x, mt, mt, mode=2, scale=30.0, margin=0.2, easy=0, eps=0.1, ignore_index=-100)
    xt = c["th"]
    sine = math.sqrt(1 - xt * xt)
    bad = f["z"].clone()
    bad[0, mt[0]] = 30.0 * (xt * c["cos_m"] - sine * c["sin_m"])
    assert R.exceeds(bad, f["z"], f["b_z"])
