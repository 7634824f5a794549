"""-m gpu: the CTC, TTS-criterion, guided-attention and speaker-head entry points of include/speecht5_b200.h called
through ctypes (speecht5_b200/_lib.py) against the fp64 statement of tests/loss_ref.py with ELEMENTWISE bounds, on
buffers laid out here with NaN sentinels everywhere the contract does not let a kernel read or write:
  - every output sits inside a NaN buffer with guard zones; padding columns of strided operands are NaN;
  - every input element the contract says is not read is NaN: CTC logits rows t >= input_lengths[b] and columns [V, ld),
    TTS inputs on masked frames (and the forced stop label), ys rows [L, Ly), label columns [L, lab_bs), attention
    columns [il, p_ld), rows beyond ol and heads >= `heads`, the x_ld / z_ld / dx_ld padding;
  - scratch (ws, sums, gsum) starts NaN, accumulated outputs start non-zero;
  - shapes sit on every launcher branch: the concurrent and sequential CTC sweeps, the CTC_GROUP tails, the gradient
    kernel at 8 / 4 / 2 / 1 warps per CTA, the TTS vector and scalar paths and the fixed-order partials loop, the
    MCE_THREADS edges.
The largest err / bound of every family is printed at the end of the module (run with -s)."""
import ctypes as C
import math

import pytest
import torch

import loss_ref as R

pytestmark = pytest.mark.gpu

NAN = float("nan")
G = 64  # guard elements before and after every buffer
REPORT = {}
F32, BF16, I64 = torch.float32, torch.bfloat16, torch.int64


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if REPORT:
        print("\nlargest err / bound per family:")
        for k in sorted(REPORT):
            print(f"  {k:44s} {REPORT[k]:.3g}")


def _lib():
    from speecht5_b200 import _lib as L
    return L.load()


def _st():
    return torch.cuda.current_stream().cuda_stream


def P(t):
    return None if t is None else C.c_void_p(t.data_ptr())


class Buf:
    """n elements inside a NaN buffer with guard zones (`off` elements past the 16-byte aligned start)."""

    def __init__(self, n, dtype=F32, fill=None, off=0):
        self.flat = torch.full((2 * G + n + off,), NAN, dtype=dtype, device="cuda")
        self.lo, self.hi = G + off, G + off + n
        self.t = self.flat[self.lo:self.hi]
        if fill is not None:
            self.t.copy_(torch.as_tensor(fill).reshape(-1).to(dtype))

    def view(self, *shape):
        return self.t.view(*shape)

    def get(self):
        return self.t.cpu()

    def untouched(self, what):
        g = torch.cat([self.flat[:self.lo], self.flat[self.hi:]]).float()
        assert bool(torch.isnan(g).all()), f"{what}: guard zone written"

    def snapshot(self):
        return self.flat.clone()

    def same_as(self, snap):
        a, b = self.flat, snap
        if a.dtype == BF16:
            a, b = a.view(torch.int16), b.view(torch.int16)
        elif a.dtype == F32:
            a, b = a.view(torch.int32), b.view(torch.int32)
        return bool(torch.equal(a, b))


def _rnd(shape, seed, scale=1.0):
    return (torch.randn(shape, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * scale).float() \
        .double()


def _ints(v):
    return torch.tensor(v, dtype=I64, device="cuda")


# ============================================================================================ CTC
def _ctc_inputs(T, B, V, tls, blank, seed, scale=1.0, repeat=False):
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(T, B, V, generator=g, dtype=torch.float64) * scale).float().double()
    labels = [k for k in range(V) if k != blank]
    tg = []
    for L in tls:
        idx = torch.randint(0, len(labels), (L,), generator=g)
        t = torch.tensor([labels[i] for i in idx], dtype=torch.long)
        if repeat and L >= 4:
            t[1], t[3] = t[0], t[2]
        tg.append(t)
    return x, tg


def run_ctc(x, tg, ils, *, blank, zi, S_max, layout="tbv", pad=3, padded_targets=False, with_grad=True):
    """One st5_ctc_loss call on NaN-guarded buffers; returns (nll, grad [T, B, V] or None, ws snapshot)."""
    lib = _lib()
    T, B, V = x.shape
    ld = V + pad
    shape = (T, B, ld) if layout == "tbv" else (B, T, ld)
    ld_t, ld_b = (B * ld, ld) if layout == "tbv" else (ld, T * ld)
    host = torch.full(shape, NAN, dtype=F32)
    for b in range(B):
        n = max(0, min(T, ils[b]))
        if layout == "tbv":
            host[:n, b, :V] = x[:n, b].float()
        else:
            host[b, :n, :V] = x[:n, b].float()
    xb = Buf(host.numel(), F32, host)
    if padded_targets:  # CTCLossPaddedFn: row b at b * S_pad, the tail filled with a valid but wrong label
        S_pad = max([len(t) for t in tg] + [1])
        flat = torch.full((B, S_pad), (blank + 1) % V, dtype=I64)
        for b, t in enumerate(tg):
            flat[b, :len(t)] = t
        offs = [b * S_pad for b in range(B)]
        flat = flat.reshape(-1)
    else:
        filler = torch.full((3,), (blank + 1) % V, dtype=I64)
        parts, offs, o = [], [], 0
        for t in tg:
            parts += [t, filler]
            offs.append(o)
            o += len(t) + 3
        flat = torch.cat(parts)
    tgt, offs_d = flat.cuda(), _ints(offs)
    il_d, tl_d = _ints(ils), _ints([len(t) for t in tg])
    nll = Buf(B)
    grad = Buf(host.numel()) if with_grad else None
    ws = Buf(int(lib.st5_ctc_ws_floats(T, B, S_max)))
    rc = lib.st5_ctc_loss(P(xb.t), ld_t, ld_b, P(tgt), P(offs_d), P(il_d), P(tl_d), P(nll.t), P(grad.t) if grad else None,
                          P(ws.t), T, B, V, S_max, blank, int(zi), _st())
    torch.cuda.synchronize()
    assert rc == 0, (rc, lib.st5_last_error())
    nll.untouched("ctc nll")
    ws.untouched("ctc ws")
    g = None
    if grad is not None:
        grad.untouched("ctc grad")
        full = grad.get().view(shape)
        assert bool(torch.isnan(full[..., V:]).all()), "ctc grad: padding columns written"
        g = full[..., :V] if layout == "tbv" else full[..., :V].transpose(0, 1)
    return nll.get(), g


def check_ctc(name, x, tg, ils, *, blank, zi, S_max, **kw):
    ref = R.ctc(x, tg, ils, blank=blank, zero_infinity=zi, S_max=S_max)
    nll, grad = run_ctc(x, tg, ils, blank=blank, zi=zi, S_max=S_max, **kw)
    fe = ref["feasible"]
    if bool(fe.any()):
        R.check(f"{name} nll", nll[fe], ref["nll"][fe], ref["b_nll"][fe], REPORT)
    want = torch.tensor([0.0 if zi else math.inf] * int((~fe).sum()), dtype=F32)
    assert torch.equal(nll[~fe], want), f"{name}: infeasible nll {nll[~fe]}"
    if grad is not None:
        R.check(f"{name} grad", grad, ref["grad"], ref["b_grad"], REPORT)
    return nll, grad, ref


def test_ctc_concurrent_and_sequential_sweeps(cuda):
    """S_max 511 / 512 take the concurrent sweeps (2 * SP <= 1024 threads), 513 / 1023 / 1024 the sequential ones: both
    run the same fp32 arithmetic, so nll is bit-identical, and each is within the bound."""
    x, tg = _ctc_inputs(560, 2, 81, [255, 120], 0, seed=1)
    ils = [560, 400]
    nlls = []
    for S_max in (511, 512, 513, 1023, 1024):
        nll, _, _ = check_ctc("ctc sweeps", x, tg, ils, blank=0, zi=False, S_max=S_max)
        nlls.append(nll)
    for n in nlls[1:]:
        assert torch.equal(n.view(torch.int32), nlls[0].view(torch.int32)), "concurrent vs sequential sweeps differ"
    # S == S_max at the top of both branches
    x, tg = _ctc_inputs(600, 1, 81, [511], 0, seed=2)
    check_ctc("ctc sweeps", x, tg, [600], blank=0, zi=False, S_max=1023)
    x, tg = _ctc_inputs(300, 1, 81, [255], 0, seed=3)
    check_ctc("ctc sweeps", x, tg, [300], blank=0, zi=False, S_max=511)


def test_ctc_group_tails_and_lengths(cuda):
    # Tn in {1, 2, 3, 4, 5, 7} (CTC_GROUP = 4 steps fetched together); target length 0; S == S_max; S > S_max;
    # input length 0 and > T
    x, tg = _ctc_inputs(9, 10, 12, [1, 1, 2, 3, 4, 5, 0, 4, 5, 2], 0, seed=4)
    ils = [1, 2, 3, 4, 5, 7, 6, 9, 9, 0]
    _, _, ref = check_ctc("ctc lengths", x, tg, ils, blank=0, zi=False, S_max=9)
    assert ref["feasible"].tolist()[6:] == [True, True, False, False]  # L = 0; S == S_max; S > S_max; length 0
    x, tg = _ctc_inputs(9, 3, 12, [3, 2, 0], 5, seed=5)
    check_ctc("ctc lengths", x, tg, [40, 9, 1000], blank=5, zi=True, S_max=7)


@pytest.mark.parametrize("zi", [False, True])
def test_ctc_repeated_labels(cuda, zi):
    # t = (a, a, b, b, c): 5 labels and 2 repeats need 7 frames; 7 is exactly feasible, 6 is not
    x, _ = _ctc_inputs(8, 3, 10, [0, 0, 0], 0, seed=6)
    t = torch.tensor([3, 3, 7, 7, 2])
    _, _, ref = check_ctc("ctc repeats", x, [t, t, t.clone()], [7, 6, 8], blank=0, zi=zi, S_max=11)
    assert ref["feasible"].tolist() == [True, False, True]


@pytest.mark.parametrize("V", [2, 31, 32, 33, 81, 1536, 1537, 6144, 12288])
def test_ctc_vocabulary_sizes(cuda, V):
    """V <= 1536: 8 warps per gradient CTA; 1537: 4; 6144: 2; 12288: 1 (48 KiB of per-symbol sums)."""
    blank = V - 1 if V % 2 else V // 2
    tl = [3, 1, 5] if V > 2 else [2, 1, 3]
    x, tg = _ctc_inputs(12, 3, V, tl, blank, seed=V)
    check_ctc("ctc V", x, tg, [12, 11, 10], blank=blank, zi=False, S_max=11)


@pytest.mark.parametrize("layout,padded", [("tbv", False), ("btv", False), ("tbv", True), ("btv", True)])
def test_ctc_layouts(cuda, layout, padded):
    x, tg = _ctc_inputs(37, 4, 40, [5, 9, 0, 12], 0, seed=7, repeat=True)
    check_ctc("ctc layout", x, tg, [37, 30, 5, 33], blank=0, zi=False, S_max=25, layout=layout, pad=5,
              padded_targets=padded)


def test_ctc_asr_bench_shape(cuda):
    """The ASR bench batch: B = 8, T = 499 frames, 160-label targets padded as CTCLossPaddedFn lays them out."""
    x, tg = _ctc_inputs(499, 8, 81, [160, 150, 140, 160, 100, 130, 160, 90], 80, seed=8)
    check_ctc("ctc asr bench", x, tg, [499, 480, 470, 499, 400, 450, 499, 300], blank=80, zi=True, S_max=321,
              pad=0, padded_targets=True)


def test_ctc_long_lattice_large_alpha(cuda):
    """700 frames, logits x 4: |alpha| reaches the thousands, where the fp32 lattice's rounding dominates the bound."""
    x, tg = _ctc_inputs(700, 2, 81, [120, 60], 0, seed=9, scale=4.0)
    _, _, ref = check_ctc("ctc long x4", x, tg, [700, 650], blank=0, zi=False, S_max=241)
    print(f"\nctc long x4: max |alpha| {ref['amax']:.4g}")
    assert ref["amax"] > 1000


# ============================================================================================ TTS loss
def run_tts(a, bf, x, ys, labels, olens, *, r, pw, g, off=(0, 0, 0)):
    """fwd + bwd with NaN on every element the kernels must not read; returns dict of host results and raw buffers."""
    lib = _lib()
    B, L, D = a.shape
    Ly, lab_w = ys.shape[1], labels.shape[1]
    valid, ol = R.tts_valid(olens, L, r)
    fr = valid[..., None]
    a_h = torch.where(fr, a, torch.full_like(a, NAN))
    b_h = torch.where(fr, bf, torch.full_like(bf, NAN))
    x_h = torch.where(valid, x, torch.full_like(x, NAN))
    y_h = torch.full((B, Ly, D), NAN, dtype=torch.float64)
    y_h[:, :L] = torch.where(fr, ys[:, :L], torch.full_like(a, NAN))
    lab_h = torch.full((B, lab_w), NAN, dtype=torch.float64)
    lab_h[:, :L] = torch.where(valid, labels[:, :L], torch.full_like(x, NAN))
    if r > 1:
        for b in range(B):
            if ol[b] >= 1:
                lab_h[b, ol[b] - 1] = NAN  # forced to 1: never read
    ab, bb = Buf(B * L * D, F32, a_h, off=off[0]), Buf(B * L * D, F32, b_h, off=off[1])
    xb, yb, lb = Buf(B * L, F32, x_h), Buf(B * Ly * D, F32, y_h, off=off[2]), Buf(B * lab_w, F32, lab_h)
    ol_d = _ints([int(o) for o in olens])
    sums = Buf(int(lib.st5_tts_loss_ws_floats(B, L)))
    out = Buf(3)
    rc = lib.st5_tts_loss_fwd(P(ab.t), P(bb.t), P(xb.t), P(yb.t), Ly * D, P(lb.t), lab_w, P(ol_d), B, L, D, r, pw,
                              P(sums.t), P(out.t), _st())
    gd = torch.tensor(g, dtype=F32, device="cuda")
    da, db, dl = Buf(B * L * D), Buf(B * L * D), Buf(B * L)
    rc2 = lib.st5_tts_loss_bwd(P(ab.t), P(bb.t), P(xb.t), P(yb.t), Ly * D, P(lb.t), lab_w, P(ol_d), P(sums.t), P(gd),
                               B, L, D, r, pw, P(da.t), P(db.t), P(dl.t), _st())
    torch.cuda.synchronize()
    assert rc == 0 and rc2 == 0, (rc, rc2, lib.st5_last_error())
    for buf, w in ((out, "out"), (sums, "sums"), (da, "d_after"), (db, "d_before"), (dl, "d_logits")):
        buf.untouched(f"tts {w}")
    return dict(out=out.get(), n=float(sums.get()[3]), d_after=da.get().view(B, L, D), d_before=db.get().view(B, L, D),
                d_logits=dl.get().view(B, L), raw=[out.snapshot(), sums.snapshot(), da.snapshot(), db.snapshot(),
                                                   dl.snapshot()], inputs=(ab, bb, xb, yb, lb, ol_d))


def _tts_inputs(B, L, D, seed, Ly=None, lab_w=None, logit_scale=2.0, exact_zero=True):
    g = torch.Generator().manual_seed(seed)
    a = (torch.randn(B, L, D, generator=g, dtype=torch.float64)).float().double()
    bf = (torch.randn(B, L, D, generator=g, dtype=torch.float64)).float().double()
    ys = (torch.randn(B, Ly or L, D, generator=g, dtype=torch.float64)).float().double()
    x = (torch.randn(B, L, generator=g, dtype=torch.float64) * logit_scale).float().double()
    labels = (torch.rand(B, lab_w or L, generator=g, dtype=torch.float64) < 0.2).double()
    if exact_zero:
        a[0, 0, : (D + 1) // 2] = ys[0, 0, : (D + 1) // 2]
    return a, bf, x, ys, labels


def check_tts(name, B, L, D, olens, r, *, pw=5.0, g=(1.0, 1.0, 1.0), seed=0, logit_scale=2.0, twice=False):
    a, bf, x, ys, labels = _tts_inputs(B, L, D, seed, Ly=L + 3, lab_w=L + 5, logit_scale=logit_scale)
    ref = R.tts_loss(a, bf, x, ys, labels, olens, r=r, pos_weight=pw, g=g)
    got = run_tts(a, bf, x, ys, labels, olens, r=r, pw=pw, g=g)
    assert got["n"] == ref["n"]
    R.check(f"tts {name} out", got["out"], ref["out"], ref["b_out"], REPORT)
    R.check(f"tts {name} d_after", got["d_after"], ref["d_after"], ref["b_d_after"], REPORT)
    R.check(f"tts {name} d_before", got["d_before"], ref["d_before"], ref["b_d_before"], REPORT)
    R.check(f"tts {name} d_logits", got["d_logits"], ref["d_logits"], ref["b_d_logits"], REPORT)
    if twice:  # same inputs, same bits (fixed-order reductions)
        again = run_tts(a, bf, x, ys, labels, olens, r=r, pw=pw, g=g)
        for u, v in zip(got["raw"], again["raw"]):
            assert torch.equal(u.view(torch.int32), v.view(torch.int32)), f"tts {name}: not bit-reproducible"
    return ref, got


@pytest.mark.parametrize("D", [1, 3, 80, 81, 132])
@pytest.mark.parametrize("r", [1, 2, 3])
def test_tts_loss_widths_and_reduction(cuda, D, r):
    # olens % r != 0, olens < r, olens == L
    check_tts(f"D{D}", 4, 41, D, [37, 40, 1 if r > 1 else 6, 41], r, g=(0.7, -1.3, 2.1), seed=D + r)


@pytest.mark.parametrize("B,L", [(1, 5), (3, 7), (5, 500)])
def test_tts_loss_row_counts(cuda, B, L):
    """B*L below 8, not a multiple of 8, and above 2,048 rows (the partials loop of the fixed-order sum)."""
    olens = [L - (b % 3) for b in range(B)]
    check_tts(f"rows{B}x{L}", B, L, 80, olens, 2, seed=B, twice=True)


def test_tts_loss_bench_shape(cuda):
    """B = 32, 626 frames, r = 2, 80 mel bins: the TTS bench batch; fwd and bwd bit-reproducible."""
    olens = [626 - 7 * b for b in range(32)]
    check_tts("bench", 32, 626, 80, olens, 2, g=(1.0, 0.0, 1.0), seed=32, twice=True)


def test_tts_loss_all_masked(cuda):
    ref, got = check_tts("all masked", 3, 9, 80, [2, 1, 0], 3, seed=3)
    assert got["n"] == 0.0 and torch.equal(got["out"], torch.zeros(3))
    for k in ("d_after", "d_before", "d_logits"):
        assert float(got[k].abs().max()) == 0.0


@pytest.mark.parametrize("pw", [1.0, 5.0])
def test_tts_loss_saturated_logits(cuda, pw):
    check_tts(f"logits30 pw{pw:g}", 3, 40, 80, [40, 33, 17], 2, pw=pw, g=(0.0, 0.0, 3.0), seed=int(pw),
              logit_scale=30.0)


# ============================================================================================ guided attention
def run_guided(att, il, ol, *, heads, T_in, p_ld, r, sigma, alpha, g, zero_rest):
    lib = _lib()
    nl = len(att)
    B, H, T_out, _ = att[0].shape
    bufs = []
    for a in att:
        h = torch.full((B, H, T_out, p_ld), NAN, dtype=torch.float64)
        for b in range(B):
            oc, ic = min(T_out, int(ol[b]) // r), min(T_in, int(il[b]))
            h[b, :heads, :oc, :ic] = a[b, :heads, :oc, :ic]
        bufs.append(Buf(h.numel(), F32, h))
    ptrs = (C.c_void_p * nl)(*[b.t.data_ptr() for b in bufs])
    il_d, ol_d = _ints([int(v) for v in il]), _ints([int(v) for v in ol])
    gsum = Buf(int(lib.st5_guided_attn_ws_floats(nl, B, heads, T_out)))
    out = Buf(1)
    rc = lib.st5_guided_attn_fwd(ptrs, nl, B, H, heads, T_out, T_in, p_ld, P(il_d), P(ol_d), r, sigma, alpha, P(gsum.t),
                                 P(out.t), _st())
    dbufs = [Buf(B * H * T_out * p_ld) for _ in range(nl)]
    dptrs = (C.c_void_p * nl)(*[b.t.data_ptr() for b in dbufs])
    gd = torch.tensor([g], dtype=F32, device="cuda")
    rc2 = lib.st5_guided_attn_bwd(dptrs, nl, B, H, heads, T_out, T_in, p_ld, P(il_d), P(ol_d), r, sigma, alpha,
                                  P(gsum.t), P(gd), zero_rest, _st())
    torch.cuda.synchronize()
    assert rc == 0 and rc2 == 0, (rc, rc2, lib.st5_last_error())
    for b in dbufs + [gsum, out]:
        b.untouched("guided")
    return dict(out=float(out.get()[0]), gsum=gsum.get()[:2], datt=[d.get().view(B, H, T_out, p_ld) for d in dbufs],
                raw=[out.snapshot(), gsum.snapshot()] + [d.snapshot() for d in dbufs])


GUIDED_CASES = [
    # n_layers, B, H, heads, T_out, T_in, p_ld, ilens, olens, r, zero_rest
    (1, 3, 4, 2, 30, 17, 20, [17, 9, 12], [60, 41, 25], 2, 0),
    (2, 3, 4, 3, 30, 17, 17, [17, 9, 12], [60, 41, 25], 2, 1),
    (3, 2, 2, 2, 25, 31, 40, [31, 40], [25, 1], 1, 1),          # ilens > T_in (clamped), one decoder step
    (4, 4, 6, 6, 14, 11, 16, [11, 5, 8, 30], [44, 2, 29, 60], 3, 0),  # olens / r == 0, olens / r > T_out, ilens > T_in
    (8, 2, 4, 1, 21, 13, 16, [13, 7], [42, 40], 2, 1),
    (2, 6, 12, 12, 180, 40, 48, [40, 31, 22, 40, 17, 9], [360, 300, 250, 180, 120, 60], 2, 0),  # > 2,048 rows
]


@pytest.mark.parametrize("case", GUIDED_CASES)
def test_guided_attention(cuda, case):
    nl, B, H, heads, T_out, T_in, p_ld, il, ol, r, zero_rest = case
    gen = torch.Generator().manual_seed(nl * 100 + B)
    att = [torch.rand(B, H, T_out, T_in, generator=gen, dtype=torch.float64).float().double() for _ in range(nl)]
    ilens, olens = torch.tensor(il), torch.tensor(ol)
    sigma, alpha, g = 0.4, 10.0, 1.7
    ref = R.guided(att, ilens, olens, r=r, heads=heads, sigma=sigma, alpha=alpha, g=g)
    got = run_guided(att, ilens, olens, heads=heads, T_in=T_in, p_ld=p_ld, r=r, sigma=sigma, alpha=alpha, g=g,
                     zero_rest=zero_rest)
    n = "guided"
    R.check(f"{n} out", torch.tensor(got["out"]), torch.tensor(ref["out"]), torch.tensor(ref["b_out"]), REPORT)
    R.check(f"{n} gsum0", got["gsum"][0], torch.tensor(ref["gsum0"]), torch.tensor(ref["b_gsum0"]), REPORT)
    assert float(got["gsum"][1]) == ref["gsum1"], "guided normaliser"
    want = torch.zeros(B, heads, T_out, p_ld, dtype=torch.float64)
    want[..., :T_in] = ref["datt"]
    bnd = torch.full_like(want, R.TINY)
    bnd[..., :T_in] = ref["b_datt"]
    for d in got["datt"]:
        R.check(f"{n} datt", d[:, :heads], want, bnd, REPORT)
        rest = d[:, heads:]
        if zero_rest:
            assert float(rest.abs().max() if rest.numel() else 0.0) == 0.0, "guided: heads >= `heads` not cleared"
        else:
            assert bool(torch.isnan(rest).all()), "guided: heads >= `heads` written without zero_rest"
    again = run_guided(att, ilens, olens, heads=heads, T_in=T_in, p_ld=p_ld, r=r, sigma=sigma, alpha=alpha, g=g,
                       zero_rest=zero_rest)
    for u, v in zip(got["raw"], again["raw"]):
        assert torch.equal(u.view(torch.int32), v.view(torch.int32)), "guided: not bit-reproducible"


# ============================================================================================ speaker head
def _strided(rows, cols, ld, dtype, fill=None):
    h = torch.full((rows, ld), NAN, dtype=torch.float64)
    if fill is not None:
        h[:, :cols] = fill
    return Buf(rows * ld, dtype, h)


def _padding_nan(buf, rows, cols, ld, what):
    full = buf.get().view(rows, ld).float()
    assert bool(torch.isnan(full[:, cols:]).all()), f"{what}: padding columns written"
    buf.untouched(what)
    return buf.get().view(rows, ld)[:, :cols]


def _spk_inputs(B, N, mode, seed):
    g = torch.Generator().manual_seed(seed)
    x = (torch.rand(B, N, generator=g, dtype=torch.float64) * 1.6 - 0.8).float().double()
    mt = torch.randint(0, N, (B,), generator=g)
    c = R.margin_consts(max(mode, 1), 30.0, 0.2)
    if B >= 6:
        x[0, mt[0]] = -0.99                   # below th = cos(pi - m)
        x[1, mt[1]] = c["th"] + 1e-3          # just above th
        x[2, mt[2]] = -1e-3                   # below 0 (easy_margin branch)
        x[3, mt[3]] = 1.0                     # |x| = 1: d sine taken as 0
        x[4, mt[4]] = -1.0
    tgt = mt.clone()
    if B >= 6:
        tgt[5] = -100                         # ignored row
        j = (int(mt[B - 1]) + 1) % N          # an exact tie at the row maximum between two non-margin columns
        k = (j + N // 2) % N if (j + N // 2) % N != int(mt[B - 1]) else (j + 1) % N
        x[B - 1, j] = x[B - 1, k] = 0.8       # (the other cosines are < 0.8)
        tgt[B - 1] = min(j, k)                # counted correct only with the lowest index
    return x.float().double(), mt, tgt        # (the fp32 values the kernel reads)


@pytest.mark.parametrize("N", [2, 5, 255, 256, 257, 1251])
@pytest.mark.parametrize("mode,easy", [(0, 0), (1, 0), (2, 0), (2, 1)])
@pytest.mark.parametrize("eps", [0.0, 0.1])
def test_margin_ce(cuda, N, mode, easy, eps):
    lib = _lib()
    B = 8 if N >= 5 else 3
    x, mt, tgt = _spk_inputs(B, N, mode, seed=N + mode)
    mtarget = mt if mode else None
    f = R.margin_ce_fwd(x, mtarget, tgt, mode=mode, scale=30.0, margin=0.2, easy=easy, eps=eps, ignore_index=-100)
    x_ld, z_ld, dx_ld = N + 3, N + 5, N + 7
    xb = _strided(B, N, x_ld, F32, x)
    zb = _strided(B, N, z_ld, F32)
    stats, lse = Buf(4 * B), Buf(B)
    mt_d = mt.cuda() if mode else None
    tg_d = tgt.cuda()
    sc = 30.0 if mode else 1.0
    rc = lib.st5_margin_ce_fwd(P(xb.t), x_ld, B, N, P(mt_d), mode, sc, 0.2, easy, P(zb.t), z_ld, P(tg_d), eps, -100,
                               P(stats.t), P(lse.t), _st())
    torch.cuda.synchronize()
    assert rc == 0, lib.st5_last_error()
    if mode == 0:
        f = R.margin_ce_fwd(x, None, tgt, mode=0, scale=1.0, margin=0.2, easy=0, eps=eps, ignore_index=-100)
    n = f"margin_ce[{mode}{'e' if easy else ''}]"
    R.check(f"{n} z", _padding_nan(zb, B, N, z_ld, n), f["z"], f["b_z"], REPORT)
    s = stats.get().view(B, 4).double()
    R.check(f"{n} loss", s[:, 0], f["loss"], f["b_loss"], REPORT)
    R.check(f"{n} nll", s[:, 1], f["nll"], f["b_nll"], REPORT)
    amb = f["ambiguous"]
    assert torch.equal(s[~amb, 2], f["correct"][~amb]), f"{n}: arg-max correctness"
    assert torch.equal(s[:, 3], f["valid"])
    v = f["valid"].bool()
    R.check(f"{n} lse", lse.get()[v], f["lse"][v], f["b_lse"][v], REPORT)
    stats.untouched(n)
    lse.untouched(n)
    # backward from the loss
    gstat = torch.tensor([0.75, -0.5], dtype=F32, device="cuda")
    dxb = _strided(B, N, dx_ld, F32)
    rc = lib.st5_margin_ce_bwd(P(xb.t), x_ld, B, N, P(mt_d), mode, sc, 0.2, easy, P(tg_d), eps, -100, P(lse.t),
                               P(gstat), None, 0, P(dxb.t), dx_ld, _st())
    torch.cuda.synchronize()
    assert rc == 0, lib.st5_last_error()
    dx, edx = R.margin_ce_bwd(f, tgt, eps=eps, ignore_index=-100, gstat=(0.75, -0.5))
    R.check(f"{n} dx", _padding_nan(dxb, B, N, dx_ld, n), dx, edx, REPORT)
    # backward from a given d z (dz_in, pitch dz_ld)
    dz = torch.randn(B, N, generator=torch.Generator().manual_seed(N), dtype=torch.float64).float().double()
    dzb = _strided(B, N, N + 2, F32, dz)
    dxb = _strided(B, N, dx_ld, F32)
    rc = lib.st5_margin_ce_bwd(P(xb.t), x_ld, B, N, P(mt_d), mode, sc, 0.2, easy, None, eps, -100, None, None,
                               P(dzb.t), N + 2, P(dxb.t), dx_ld, _st())
    torch.cuda.synchronize()
    assert rc == 0, lib.st5_last_error()
    dx, edx = R.margin_ce_bwd(f, None, eps=eps, ignore_index=-100, dz_in=dz)
    R.check(f"{n} dx (dz_in)", _padding_nan(dxb, B, N, dx_ld, n), dx, edx, REPORT)


def test_margin_ce_target_out_of_range_gives_nan(cuda):
    lib = _lib()
    B, N = 3, 7
    x = torch.rand(B, N, dtype=torch.float64)
    xb = Buf(B * N, F32, x)
    tg = _ints([2, N, -3])
    stats, lse = Buf(4 * B), Buf(B)
    rc = lib.st5_margin_ce_fwd(P(xb.t), N, B, N, None, 0, 1.0, 0.0, 0, None, N, P(tg), 0.1, -100, P(stats.t), P(lse.t),
                               _st())
    torch.cuda.synchronize()
    assert rc == 0
    s = stats.get().view(B, 4)
    assert bool(torch.isfinite(s[0]).all())
    for b in (1, 2):
        assert math.isnan(s[b, 0]) and math.isnan(s[b, 1]) and s[b, 2] == 0 and s[b, 3] == 1


@pytest.mark.parametrize("E", [1, 33, 768])
@pytest.mark.parametrize("dts", ["f32", "bf16"])
def test_l2norm_rows(cuda, E, dts):
    lib = _lib()
    dt = F32 if dts == "f32" else BF16
    u = R.U32 if dt == F32 else R.U_BF16
    rows = 37
    x = torch.randn(rows, E, generator=torch.Generator().manual_seed(E), dtype=torch.float64).to(dt).double()
    x[5] = 0.0          # clamped row (norm 0)
    x[6] = 1e-14        # clamped row (norm < 1e-12)
    x = x.to(dt).double()
    x_ld = E + 3
    xb = _strided(rows, E, x_ld, dt, x)
    y, nrm = Buf(rows * E), Buf(rows)
    rc = lib.st5_l2norm_rows_fwd(P(xb.t), x_ld, int(dt == BF16), P(y.t), P(nrm.t), rows, E, _st())
    torch.cuda.synchronize()
    assert rc == 0, lib.st5_last_error()
    f = R.l2norm_fwd(x)
    n = f"l2norm_fwd[{dts}]"
    R.check(f"{n} y", y.get().view(rows, E), f["y"], f["b_y"], REPORT)
    R.check(f"{n} nrm", nrm.get(), f["nrm"], f["b_nrm"], REPORT)
    y.untouched(n)
    nrm.untouched(n)
    # backward from the kernel's own y / nrm
    yk, nk = y.get().view(rows, E).double(), nrm.get().double()
    dy = torch.randn(rows, E, generator=torch.Generator().manual_seed(E + 1), dtype=torch.float64).float().double()
    dyb = Buf(rows * E, F32, dy)
    ref, bnd = R.l2norm_bwd(dy, yk, nk)
    for acc in ([0, 1] if dt == F32 else [0]):
        dx_ld = E + 5
        init = torch.randn(rows, E, generator=torch.Generator().manual_seed(3), dtype=torch.float64).float().double()
        dxb = _strided(rows, E, dx_ld, dt, init if acc else None)
        rc = lib.st5_l2norm_rows_bwd(P(dyb.t), P(y.t), P(nrm.t), P(dxb.t), dx_ld, int(dt == BF16), acc, rows, E, _st())
        torch.cuda.synchronize()
        assert rc == 0, lib.st5_last_error()
        want = ref + (init if acc else 0.0)
        R.check(f"l2norm_bwd[{dts}]{' +=' if acc else ''}", _padding_nan(dxb, rows, E, dx_ld, "l2norm_bwd"), want,
                bnd + (R.U32 * want.abs() if acc else 0.0) + u * want.abs(), REPORT)


@pytest.mark.parametrize("T", [1, 7, 8000])
@pytest.mark.parametrize("dts", ["f32", "bf16"])
def test_time_mean(cuda, T, dts):
    lib = _lib()
    dt = F32 if dts == "f32" else BF16
    u = R.U32 if dt == F32 else R.U_BF16
    B, Cc = 3, 37
    x = (torch.randn(B, T, Cc, generator=torch.Generator().manual_seed(T), dtype=torch.float64) + 0.3).to(dt).double()
    xb, y = Buf(B * T * Cc, dt, x), Buf(B * Cc, dt)
    rc = lib.st5_time_mean_fwd(P(xb.t), P(y.t), int(dt == BF16), B, T, Cc, _st())
    torch.cuda.synchronize()
    assert rc == 0, lib.st5_last_error()
    ref, bnd = R.time_mean_fwd(x.view(B, T, Cc), u)
    R.check(f"time_mean_fwd[{dts}]", y.get().view(B, Cc), ref, bnd, REPORT)
    y.untouched("time_mean_fwd")
    dy = torch.randn(B, Cc, generator=torch.Generator().manual_seed(T + 1), dtype=torch.float64).to(dt).double()
    dyb, dx = Buf(B * Cc, dt, dy), Buf(B * T * Cc, dt)
    rc = lib.st5_time_mean_bwd(P(dyb.t), P(dx.t), int(dt == BF16), B, T, Cc, _st())
    torch.cuda.synchronize()
    assert rc == 0, lib.st5_last_error()
    ref, bnd = R.time_mean_bwd(dy, T, u)
    R.check(f"time_mean_bwd[{dts}]", dx.get().view(B, T, Cc), ref, bnd, REPORT)
    dx.untouched("time_mean_bwd")


# ============================================================================================ rejections
def _rejected(rc, bufs, what):
    torch.cuda.synchronize()
    assert rc in (-2, -3), f"{what}: returned {rc}"
    for b, snap in bufs:
        assert b.same_as(snap), f"{what}: a buffer changed on a rejected call"
    return rc


def test_rejections_leave_every_buffer_unchanged(cuda):
    lib = _lib()
    st = _st()

    def snap(*bufs):
        return [(b, b.snapshot()) for b in bufs]

    # ---- CTC: argument checks, and V > 12288 with a gradient (checked before any launch)
    T, B, V = 4, 2, 12289
    xb = Buf(T * B * V, F32, torch.randn(T * B * V))
    tg, offs, il, tl = _ints([1, 2, 3, 4]), _ints([0, 2]), _ints([4, 4]), _ints([2, 2])
    nll, grad, ws = Buf(B), Buf(T * B * V), Buf(int(lib.st5_ctc_ws_floats(T, B, 5)))
    bufs = snap(xb, nll, grad, ws)
    args = dict(T=T, B=B, V=V, S_max=5, blank=0)
    for bad in (dict(), dict(T=0), dict(B=0), dict(V=0, blank=0), dict(S_max=0), dict(S_max=1025), dict(blank=-1),
                dict(blank=V)):
        a = {**args, **bad}  # (no override: V = 12289 > 12288 with a gradient)
        rc =lib.st5_ctc_loss(P(xb.t), B * V, V, P(tg), P(offs), P(il), P(tl), P(nll.t), P(grad.t), P(ws.t), a["T"],
                              a["B"], a["V"], a["S_max"], a["blank"], 0, st)
        assert _rejected(rc, bufs, f"ctc {bad or 'V=12289'}") == -2

    # ---- TTS loss: sizes, and the float4 path's alignment (D % 4 == 0)
    B, L, D = 2, 5, 8
    n = B * L * D
    a, bb, ys = Buf(n + 4, F32, torch.randn(n + 4)), Buf(n + 4, F32, torch.randn(n + 4)), Buf(n + 8, F32, torch.randn(n + 8))
    lg, lab = Buf(B * L, F32, torch.randn(B * L)), Buf(B * L, F32, torch.zeros(B * L))
    ol = _ints([5, 3])
    sums, out = Buf(int(lib.st5_tts_loss_ws_floats(B, L))), Buf(3)
    da, db, dl = Buf(n + 4), Buf(n + 4), Buf(B * L)
    gd = torch.ones(3, device="cuda")
    bufs = snap(a, bb, ys, lg, lab, sums, out, da, db, dl)
    base = dict(a=a.t, b=bb.t, y=ys.t, y_bs=L * D, B=B, L=L, D=D, r=1, da=da.t, db=db.t)
    off1 = lambda t: t[1:]  # noqa: E731  (4 bytes past a 16-byte boundary)
    cases = [dict(B=0), dict(L=0), dict(D=0), dict(r=0), dict(a=off1(a.t)), dict(b=off1(bb.t)), dict(y=off1(ys.t)),
             dict(y_bs=L * D + 2)]
    for bad in cases + [dict(da=off1(da.t)), dict(db=off1(db.t))]:
        c = {**base, **bad}
        if "da" not in bad and "db" not in bad:
            rc = lib.st5_tts_loss_fwd(P(c["a"]), P(c["b"]), P(lg.t), P(c["y"]), c["y_bs"], P(lab.t), L, P(ol), c["B"],
                                      c["L"], c["D"], c["r"], 5.0, P(sums.t), P(out.t), st)
            assert _rejected(rc, bufs, f"tts_loss_fwd {bad}") == -2
        rc = lib.st5_tts_loss_bwd(P(c["a"]), P(c["b"]), P(lg.t), P(c["y"]), c["y_bs"], P(lab.t), L, P(ol), P(sums.t),
                                  P(gd), c["B"], c["L"], c["D"], c["r"], 5.0, P(c["da"]), P(c["db"]), P(dl.t), st)
        assert _rejected(rc, bufs, f"tts_loss_bwd {bad}") == -2

    # ---- guided attention
    nl, B, H, T_out, T_in = 2, 2, 2, 6, 5
    att = [Buf(B * H * T_out * T_in, F32, torch.rand(B * H * T_out * T_in)) for _ in range(nl)]
    datt = [Buf(B * H * T_out * T_in) for _ in range(nl)]
    aptr = (C.c_void_p * nl)(*[t.t.data_ptr() for t in att])
    dptr = (C.c_void_p * nl)(*[t.t.data_ptr() for t in datt])
    il, ol = _ints([5, 3]), _ints([12, 8])
    gsum, out = Buf(int(lib.st5_guided_attn_ws_floats(8, B, H, T_out)) + 8), Buf(1)
    bufs = snap(*att, *datt, gsum, out)
    base = dict(nl=nl, B=B, H=H, heads=H, T_out=T_out, T_in=T_in, p_ld=T_in, r=2, sigma=0.4)
    for bad in (dict(nl=0), dict(nl=9), dict(B=0), dict(H=0, heads=0), dict(heads=0), dict(heads=H + 1),
                dict(T_out=0), dict(T_in=0), dict(p_ld=T_in - 1), dict(r=0), dict(sigma=0.0), dict(sigma=NAN)):
        c = {**base, **bad}
        args = (c["nl"], c["B"], c["H"], c["heads"], c["T_out"], c["T_in"], c["p_ld"], P(il), P(ol), c["r"], c["sigma"],
                10.0)
        rc = lib.st5_guided_attn_fwd(aptr, *args, P(gsum.t), P(out.t), st)
        assert _rejected(rc, bufs, f"guided_attn_fwd {bad}") == -2
        rc = lib.st5_guided_attn_bwd(dptr, *args, P(gsum.t), P(gd), 1, st)
        assert _rejected(rc, bufs, f"guided_attn_bwd {bad}") == -2

    # ---- l2norm
    rows, E = 4, 8
    x = Buf(rows * E, F32, torch.randn(rows * E))
    y, nrm = Buf(rows * E, F32, torch.randn(rows * E)), Buf(rows, F32, torch.rand(rows) + 1)
    dx = Buf(rows * E)
    bufs = snap(x, y, nrm, dx)
    for bad, code in ((dict(rows=-1), -2), (dict(E=0), -2), (dict(ld=E - 1), -2), (dict(dtype=2), -2)):
        c = {**dict(rows=rows, E=E, ld=E, dtype=0), **bad}
        rc = lib.st5_l2norm_rows_fwd(P(x.t), c["ld"], c["dtype"], P(y.t), P(nrm.t), c["rows"], c["E"], st)
        assert _rejected(rc, bufs, f"l2norm_fwd {bad}") == code
        rc = lib.st5_l2norm_rows_bwd(P(y.t), P(y.t), P(nrm.t), P(dx.t), c["ld"], c["dtype"], 0, c["rows"], c["E"], st)
        assert _rejected(rc, bufs, f"l2norm_bwd {bad}") == code
    rc = lib.st5_l2norm_rows_bwd(P(y.t), P(y.t), P(nrm.t), P(dx.t), E, 1, 1, rows, E, st)  # accumulate into bf16
    assert _rejected(rc, bufs, "l2norm_bwd accumulate bf16") == -3

    # ---- margin + CE
    B, N = 3, 6
    x = Buf(B * N, F32, torch.rand(B * N))
    z, stats, lse = Buf(B * N), Buf(4 * B), Buf(B, F32, torch.zeros(B))
    dxm, dz = Buf(B * N), Buf(B * N, F32, torch.randn(B * N))
    mt, tg = _ints([0, 1, 2]), _ints([0, 1, 2])
    gs = torch.ones(2, device="cuda")
    bufs = snap(x, z, stats, lse, dxm, dz)
    fb = dict(B=B, N=N, mt=mt, mode=2, x_ld=N, z=z.t, z_ld=N, tg=tg, stats=stats.t, lse=lse.t)
    for bad in (dict(B=-1), dict(mode=3), dict(N=1), dict(x_ld=N - 1), dict(z_ld=N - 1), dict(mode=0),
                dict(stats=None), dict(lse=None)):
        c = {**fb, **bad}
        rc = lib.st5_margin_ce_fwd(P(x.t), c["x_ld"], c["B"], c["N"], P(c["mt"]), c["mode"], 30.0, 0.2, 0, P(c["z"]),
                                   c["z_ld"], P(c["tg"]), 0.1, -100, P(c["stats"]), P(c["lse"]), st)
        assert _rejected(rc, bufs, f"margin_ce_fwd {bad}") == -2
    bb_ = dict(B=B, N=N, mt=mt, mode=2, x_ld=N, tg=tg, lse=lse.t, gs=gs, dz=None, dz_ld=N, dx_ld=N)
    for bad in (dict(B=-1), dict(mode=3), dict(N=1), dict(x_ld=N - 1), dict(dx_ld=N - 1), dict(mode=0),
                dict(dz=dz.t), dict(tg=None), dict(lse=None), dict(gs=None), dict(tg=None, dz=dz.t, dz_ld=N - 1)):
        c = {**bb_, **bad}
        rc = lib.st5_margin_ce_bwd(P(x.t), c["x_ld"], c["B"], c["N"], P(c["mt"]), c["mode"], 30.0, 0.2, 0, P(c["tg"]),
                                   0.1, -100, P(c["lse"]), P(c["gs"]), P(c["dz"]), c["dz_ld"], P(dxm.t), c["dx_ld"], st)
        assert _rejected(rc, bufs, f"margin_ce_bwd {bad}") == -2

    # ---- time mean
    B, T, Cc = 2, 3, 5
    x = Buf(B * T * Cc, F32, torch.randn(B * T * Cc))
    y, dx = Buf(B * Cc), Buf(B * T * Cc)
    bufs = snap(x, y, dx)
    for bad in (dict(B=-1), dict(T=0), dict(C=0), dict(dtype=2)):
        c = {**dict(B=B, T=T, C=Cc, dtype=0), **bad}
        rc = lib.st5_time_mean_fwd(P(x.t), P(y.t), c["dtype"], c["B"], c["T"], c["C"], st)
        assert _rejected(rc, bufs, f"time_mean_fwd {bad}") == -2
        rc = lib.st5_time_mean_bwd(P(y.t), P(dx.t), c["dtype"], c["B"], c["T"], c["C"], st)
        assert _rejected(rc, bufs, f"time_mean_bwd {bad}") == -2
