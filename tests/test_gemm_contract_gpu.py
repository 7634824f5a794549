"""-m gpu: st5_gemm_bf16 (csrc/gemm.cu) against its contract in include/speecht5_b200.h, stated in fp64 by
tests/gemm_emulator.gemm on CPU copies of the same operands, with ELEMENTWISE bounds (one wrong 32 x 32 block, a dropped
k-block or one wrong mask bit fails), NaN sentinels around every output and in every operand's padding, and dropout
masks compared bit for bit with tests/dropout_ref.py. The test_core_window_* cases hand the kernel the overlapping
window operands of the convolutions (ld < K, or ld < rows MN-major), with NaN right after the last element a window
reads.

The tile width (128 x 64 or 128 x 128) is chosen by a cost model once per call and ST5_GEMM_BN pins it for a whole
process, so the test_core_* cases run here with the cost model's choice and again in two child processes with each
width pinned (test_core_cases_under_both_pinned_tile_widths)."""
import math
import os
import subprocess
import sys

import pytest
import torch

import dropout_ref as D
import gemm_emulator as E

pytestmark = pytest.mark.gpu

NAN = float("nan")
# Elementwise bound of the fp32-accumulated product: |got - ref| <= C_ACC * 2^-24 * sqrt(K) * (|A| @ |B|^T). The tensor
# cores add bf16 x bf16 products (exact in fp32) into fp32 accumulators; rounding errors of a K-term fp32 sum grow like
# sqrt(K) * 2^-24 * sum|a b| when they are unbiased. C_ACC = 16 leaves room for the tail of that distribution and for the
# tensor-core adder's truncating alignment, while one wrong product term (|a b| ~ 1 / sqrt(K) of the magnitude) or one
# wrong block still exceeds it by orders of magnitude.
C_ACC = 16.0
TINY = 2.0 ** -40


def _r8(x):
    return (x + 7) // 8 * 8


class Operand:
    """bf16 operand [nb2][nb1] x rows x K stored K-major ([rows][ld]) or MN-major ([K][ld]) inside a NaN-filled buffer:
    the padding columns / rows up to ld and the gaps between padded batch entries are NaN, so reading them poisons the
    product."""

    def __init__(self, rows, K, mn, nb1=1, nb2=1, bcast1=False, bcast2=False, gen=None, scale=1.0, dev="cuda",
                 lay=None):
        if lay is not None:
            self._recorded(rows, K, mn, nb1, nb2, lay, gen, scale, dev)
            return
        ext = rows if mn else K
        self.ld = _r8(ext) + 8
        inner = (K if mn else rows) * self.ld
        self.bs1 = 0 if (bcast1 or nb1 == 1) else inner + 16
        self.bs2 = 0 if (bcast2 or nb2 == 1) else (self.bs1 * nb1 if self.bs1 else inner) + 24
        size = (nb2 - 1) * self.bs2 + (nb1 - 1) * self.bs1 + inner + 64
        buf = torch.full((size,), NAN, dtype=torch.float32)
        outer = K if mn else rows
        for b2 in range(nb2 if self.bs2 else 1):
            for b1 in range(nb1 if self.bs1 else 1):
                o = b2 * self.bs2 + b1 * self.bs1
                v = torch.randn(outer, ext, generator=gen) * scale
                buf[o:o + inner].view(outer, self.ld)[:, :ext] = v
        self.cpu = buf.to(torch.bfloat16)
        self.dev = self.cpu.to(dev)
        self.mn = mn

    def _recorded(self, rows, K, mn, nb1, nb2, lay, gen, scale, dev):
        """lay = (ld, bs1, bs2, off): a layout taken from a real launch (overlapping batch entries, interleaved heads or
        windows included). Every element the operand covers is random, everything else NaN; the operand starts `off`
        elements past a 128-byte boundary, after a NaN guard zone."""
        self.ld, self.bs1, self.bs2, off = lay
        self.mn = mn
        outer, inner = (K, rows) if mn else (rows, K)
        o = 64 + off
        idx = (o + torch.arange(nb2)[:, None, None, None] * self.bs2 + torch.arange(nb1)[None, :, None, None] * self.bs1
               + torch.arange(outer)[:, None] * self.ld + torch.arange(inner)).reshape(-1)
        buf = torch.full((int(idx.max()) + 65,), NAN, dtype=torch.float32)
        buf[idx] = torch.randn(idx.numel(), generator=gen) * scale
        buf = buf.to(torch.bfloat16)
        self.cpu = buf[o:]
        self.dev = buf.to(dev)[o:]

    def kw(self, which):
        return {f"{which}_mn": self.mn, f"{which}_ld": self.ld, f"{which}_bs": (self.bs1, self.bs2)}


class WindowOperand(Operand):
    """bf16 operand rows x K read as an overlapping window, the layout of the convolutions: K-major with ld < K (row r
    is the K elements from r * ld) or MN-major with ld < rows (k-row k is the rows elements from k * ld). The memory
    past the logical K of a row (past `rows` of a k-row) is valid data of the next rows, finite; the zero fill of the
    TMA map (dims[0] = K, or rows) alone keeps it out of a ragged last block. NaN starts right after the last element
    a window may read, (rows - 1) ld + K (MN-major: (K - 1) ld + rows), and fills the gap between batch entries."""

    def __init__(self, rows, K, mn, ld, nb1=1, gen=None, scale=1.0, dev="cuda"):
        assert ld < (rows if mn else K), "not an overlapping window"
        span = (K - 1) * ld + rows if mn else (rows - 1) * ld + K
        self.ld, self.mn = ld, mn
        self.bs1 = 0 if nb1 == 1 else _r8(span) + 16
        self.bs2 = 0
        buf = torch.full(((nb1 - 1) * self.bs1 + span + 64,), NAN, dtype=torch.float32)
        for b1 in range(nb1):
            buf[b1 * self.bs1:b1 * self.bs1 + span] = torch.randn(span, generator=gen) * scale
        self.cpu = buf.to(torch.bfloat16)
        self.dev = self.cpu.to(dev)


class OutLayout:
    """Logical [nb2][nb1][M][N] region at pitch c_ld inside a larger buffer (rows past M, columns past N, gaps between
    batch entries and guard zones before and after); `inside` marks the logical elements."""

    def __init__(self, M, N, nb1=1, nb2=1, c_ld=None, shared=False, misalign=0, bs=None):
        """bs: batch strides taken from a real launch (interleaved heads or a shared output included)."""
        self.M, self.N, self.nb1, self.nb2 = M, N, nb1, nb2
        self.c_ld = c_ld if c_ld is not None else _r8(N) + 8
        self.bs1 = 0 if (shared or nb1 == 1) else (M + 3) * self.c_ld
        self.bs2 = 0 if (shared or nb2 == 1) else (self.bs1 * nb1 if self.bs1 else (M + 3) * self.c_ld) + 8 * self.c_ld
        if bs is not None:
            self.bs1, self.bs2 = bs
        self.base = 32 + misalign
        b2 = torch.arange(nb2)[:, None, None, None] * self.bs2
        b1 = torch.arange(nb1)[None, :, None, None] * self.bs1
        idx = self.base + b2 + b1 + torch.arange(M)[:, None] * self.c_ld + torch.arange(N)
        self.idx = idx  # [nb2, nb1, M, N] flat positions
        self.size = max(self.base + (nb2 - 1) * self.bs2 + (nb1 - 1) * self.bs1 + (M + 3) * self.c_ld,
                        int(idx.max()) + 1) + 64
        self.inside = torch.zeros(self.size, dtype=torch.bool)
        self.inside[idx.reshape(-1)] = True

    def kw(self):
        return dict(c_ld=self.c_ld, c_bs=(self.bs1, self.bs2))

    def buffer(self, dtype, fill=None, gen=None, scale=1.0):
        """NaN everywhere; the logical region random (fill='randn') or zero (fill='zero') if asked."""
        buf = torch.full((self.size,), NAN, dtype=torch.float32)
        if fill == "randn":
            buf[self.idx.reshape(-1)] = torch.randn(self.idx.numel(), generator=gen) * scale
        elif fill == "zero":
            buf[self.idx.reshape(-1)] = 0.0
        return buf.to(dtype)

    def region(self, buf):
        return buf[self.idx]

    def assert_outside_untouched(self, got, what="output"):
        bad = ~torch.isnan(got[~self.inside].float())
        assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements written outside [M) x [N) (first at " \
                                    f"{int(torch.nonzero(~self.inside)[bad.nonzero()[0]])})"


def _act_f64(v, act):
    return E._act(v, act)


def run_gemm(M, N, K, *, a_mn=False, b_mn=False, nb1=1, nb2=1, a_bcast=(False, False), b_bcast=(False, False),
             out_dtype=torch.float32, c_ld=None, shared=False, misalign=0, alpha=1.0, accumulate=0, bias=None,
             bias2_rows=0, residual=False, c_pre=False, act=None, actgrad_act=None, drop_p=0.0, seed=1234,
             offset=7, device_seed=False, operand_scale=None, seed_data=0, check=True, a_win=None, b_win=None,
             a_lay=None, b_lay=None, c_bs=None, residual_is_out=False, blocks=None, bias2_off=0, dev="cuda"):
    """Run K.gemm on NaN-guarded buffers, then compare with the fp64 statement elementwise. Returns a dict of the CPU
    results (got / ref regions, pre-activation, keep mask) for case-specific checks. a_win / b_win: the row pitch of
    an overlapping-window operand (WindowOperand, nb2 = 1).

    A launch recorded from a real update is replayed with its own layout: a_lay / b_lay = (ld, bs1, bs2, element
    offset from a 16-byte boundary), c_ld / c_bs / misalign for the output (c_pre, residual and actgrad_pre share its
    layout), residual_is_out for an in-place residual (residual = out), bias and bias2_off element offsets. blocks: a list of (rows, cols) index tensors (None: all) -- the fp64
    statement is evaluated and compared on those outputs only (every batch entry, full K); the sentinels are checked
    everywhere."""
    from speecht5_b200 import kernels as K_
    dev = torch.device(dev)
    gen = torch.Generator().manual_seed(seed_data)
    # operand scale: the pre-activation has unit standard deviation whatever K is
    sc = operand_scale if operand_scale is not None else K ** -0.25
    A = WindowOperand(M, K, a_mn, a_win, nb1, gen=gen, scale=sc, dev=dev) if a_win else \
        Operand(M, K, a_mn, nb1, nb2, *a_bcast, gen=gen, scale=sc, dev=dev, lay=a_lay)
    B = WindowOperand(N, K, b_mn, b_win, nb1, gen=gen, scale=sc, dev=dev) if b_win else \
        Operand(N, K, b_mn, nb1, nb2, *b_bcast, gen=gen, scale=sc, dev=dev, lay=b_lay)
    L = OutLayout(M, N, nb1, nb2, c_ld=c_ld, shared=shared, misalign=misalign, bs=c_bs)
    c0 = L.buffer(out_dtype, fill="randn" if (accumulate == 1 or residual_is_out) else
                  ("zero" if accumulate == 2 else None), gen=gen)
    if accumulate == 2 and shared:
        c0[L.idx[0, 0].reshape(-1)] = torch.randn(M * N, generator=gen).to(out_dtype)
    elif accumulate == 2 and c_bs is not None:  # a recorded reduce-add: the output starts non-zero
        c0[L.idx.reshape(-1)] = torch.randn(L.idx.numel(), generator=gen).to(out_dtype)
    # bias / bias2: CPU views for the fp64 statement, and device views at the same element offset into a buffer that
    # is copied whole (a copy of the view alone would start 16-byte aligned again)
    bias_t = bias2_t = bias_d = bias2_d = None
    if bias is not None:
        bb = torch.randn(N + 8, generator=gen)
        o = 1 if bias == "offset" else (0 if bias == "aligned" else bias)  # "offset": 4 bytes past a 16-byte boundary
        bias_t, bias_d = bb[o:N + o], bb.to(dev)[o:N + o]
    if bias2_rows:
        n2 = (M + bias2_rows - 1) // bias2_rows
        b2 = torch.randn(n2 * N + 8, generator=gen)
        bias2_t, bias2_d = (t[bias2_off:bias2_off + n2 * N].view(n2, N) for t in (b2, b2.to(dev)))
    res_t = c0 if residual_is_out else (L.buffer(out_dtype, fill="randn", gen=gen) if residual else None)
    ag_t = None
    if actgrad_act is not None:
        ag_t = L.buffer(out_dtype, fill="randn", gen=gen, scale=0.7)
        ag_t = torch.where(ag_t.float().abs() > 2, ag_t.float().sign() * 2, ag_t.float()).to(out_dtype)
    pre_t = L.buffer(out_dtype) if c_pre else None
    common = dict(M=M, N=N, K=K, nb1=nb1, nb2=nb2, alpha=alpha, accumulate=accumulate, act=act, drop_p=drop_p,
                  **A.kw("a"), **B.kw("b"), **L.kw())

    def dv(t):
        return None if t is None else t.to(dev)
    # ---- device run
    cd = c0.to(dev, copy=True)  # (a copy on the CPU too: c0 is the reference's starting point)
    out_d = cd[L.base:]
    if residual_is_out:
        res_d = cd
    kseed, koff = seed, offset
    if device_seed:
        seed_buf = torch.tensor([seed], dtype=torch.int64, device=dev)
        kseed, koff = seed_buf.data_ptr(), offset | (1 << 63)
    pre_d = dv(pre_t)
    if not residual_is_out:
        res_d = dv(res_t)
    ag_d = dv(ag_t)
    K_.gemm(A.dev, B.dev, out_d, **common, bias=bias_d, bias2=bias2_d, bias2_rows=bias2_rows,
            residual=None if res_d is None else res_d[L.base:], c_pre=None if pre_d is None else pre_d[L.base:],
            actgrad_pre=None if ag_d is None else ag_d[L.base:], actgrad_act=actgrad_act, seed=kseed, offset=koff)
    if dev.type == "cuda":
        torch.cuda.synchronize()
    got = cd.cpu()
    got_pre = pre_d.cpu() if pre_d is not None else None
    # ---- fp64 statement
    ref = c0.clone()
    ref_pre = L.buffer(out_dtype) if c_pre else None
    # exact pre-activation v + c_old + bias + bias2, and |alpha| |A| |B|^T, in fp64
    pre64 = c0.double() if accumulate == 1 else L.buffer(torch.float64, fill="zero")
    plain = dict(common, act=None, drop_p=0.0, accumulate=1 if accumulate == 1 else 0)
    mag = L.buffer(torch.float32, fill="zero")
    magkw = dict(plain, alpha=abs(alpha), accumulate=2 if accumulate == 2 else 0)
    a_abs, b_abs = A.cpu.float().abs().to(torch.bfloat16), B.cpu.float().abs().to(torch.bfloat16)
    sel, parts = None, [(None, None)]  # the outputs compared (all, or the union of the blocks), as disjoint parts
    if blocks:
        sel = torch.zeros(nb2, nb1, M, N, dtype=torch.bool)
        for rows, cols in blocks:
            sel[:, :, slice(None) if rows is None else rows[:, None], slice(None) if cols is None else cols] = True
        pattern, which = torch.unique(sel[0, 0], dim=0, return_inverse=True)  # rows with the same columns: one part
        parts = [((which == i).nonzero()[:, 0], p.nonzero()[:, 0]) for i, p in enumerate(pattern) if p.any()]
    for rows, cols in parts:  # (disjoint: accumulating statements must see every output once)
        E.gemm(A.cpu, B.cpu, ref[L.base:], **common, bias=bias_t, bias2=bias2_t, bias2_rows=bias2_rows,
               residual=None if res_t is None else res_t[L.base:], c_pre=None if ref_pre is None else ref_pre[L.base:],
               actgrad_pre=None if ag_t is None else ag_t[L.base:], actgrad_act=actgrad_act, seed=seed, offset=offset,
               rows=rows, cols=cols)
        if accumulate != 2:
            E.gemm(A.cpu, B.cpu, pre64[L.base:], **plain, bias=bias_t, bias2=bias2_t, bias2_rows=bias2_rows,
                   rows=rows, cols=cols)
        E.gemm(a_abs, b_abs, mag[L.base:], **magkw, rows=rows, cols=cols)

    def region(buf):
        x = L.region(buf)
        return x if sel is None else x[sel]
    r = dict(L=L, got=region(got).double(), ref=region(ref).double(), pre=region(pre64).double(),
             mag=region(mag).double(), got_buf=got, ref_buf=ref, got_pre=got_pre, ref_pre=ref_pre, sel=sel)
    if drop_p > 0:
        if sel is None:
            r["keep"] = E.gemm_keep(M, N, nb1 * nb2, drop_p, seed, offset).reshape(nb2, nb1, M, N)
        else:
            import numpy as np
            z, m, n = (t.numpy().astype(np.uint64) for t in (sel.reshape(-1, M, N).nonzero().T))
            r["keep"] = torch.from_numpy(D.keep_mask(seed, offset, (z * np.uint64(M) + m) * np.uint64(N) + n, drop_p))
    if not check:
        return r
    # ---- bound
    scale = D.drop_scale(drop_p) if drop_p > 0 else 1.0
    agmax = 1.0
    if ag_t is not None:
        agp = region(ag_t).double()
        agmax = float(agp.abs().max()) if actgrad_act == "gate" else 1.2
    amp = 1.2 * scale * agmax
    addmag = r["pre"].abs()
    if accumulate in (1, 2):
        addmag = addmag + region(c0).double().abs()
    bound = C_ACC * 2.0 ** -24 * math.sqrt(K) * r["mag"] * amp + 2.0 ** -20 * addmag * amp + TINY
    if act in ("gelu_tanh", "gelu_tanh_gate"):  # MUFU tanh.approx: |error| <= 2^-11 |tanh|
        bound = bound + 2.0 ** -10 * (1 + r["pre"].abs()) * scale * agmax
    if actgrad_act == "gelu_tanh":  # act'(pre) through the same approximate tanh
        v = _act_f64(r["pre"], act).abs() * scale
        bound = bound + 2.0 ** -8 * v
    if res_t is not None:
        bound = bound + 2.0 ** -22 * region(res_t).double().abs()
    if out_dtype == torch.bfloat16:  # got and ref are both rounded to bf16: one unit in the last place apart at most
        bound = bound + 2.0 ** -7 * r["ref"].abs()
    err = (r["got"] - r["ref"]).abs()
    bad = ~(err <= bound)
    r["worst"] = float((err / bound).nan_to_num(math.inf).max()) if err.numel() else 0.0
    if bool(bad.any()):
        first = bad.nonzero()[0] if sel is None else sel.nonzero()[int(bad.nonzero()[0])]
        raise AssertionError(f"{int(bad.sum())} of {bad.numel()} outputs off; first (b2, b1, m, n) = "
                             f"{tuple(int(i) for i in first)}, max err/bound {r['worst']:.3g}")
    L.assert_outside_untouched(got)
    if sel is not None:  # outputs outside the compared blocks: written at least
        unwritten = ~torch.isfinite(L.region(got).float())
        assert not bool(unwritten.any()), f"output (b2, b1, m, n) = {tuple(int(i) for i in unwritten.nonzero()[0])} " \
                                          "not written"
    if c_pre:
        L.assert_outside_untouched(got_pre, "c_pre")
        if act != "gelu_tanh_gate":  # the pre-activation itself
            pb = C_ACC * 2.0 ** -24 * math.sqrt(K) * r["mag"] * 1.2 + 2.0 ** -20 * addmag + TINY
            if out_dtype == torch.bfloat16:
                pb = pb + 2.0 ** -8 * r["pre"].abs()
            e = (region(got_pre).double() - r["pre"]).abs()
            assert bool((e <= pb).all()), f"c_pre off at {tuple(int(i) for i in (e > pb).nonzero()[0])}"
    if drop_p > 0:
        before = _act_f64(r["pre"], act)
        sure = before.abs() > 1e-3
        if res_t is None and ag_t is None:
            kept = r["got"] != 0
            assert torch.equal(kept[sure], r["keep"][sure]), "dropout mask differs from dropout_ref"
    return r


MAJORS = [(False, False), (False, True), (True, False), (True, True)]
MAJOR_IDS = ["kk", "km", "mk", "mm"]
SHAPES = [(1, 8, 8), (77, 40, 24), (128, 128, 64), (300, 200, 200), (513, 328, 1000), (256, 256, 3072),
          (2048, 1536, 136), (150, 333, 72), (90, 330, 40)]


# ------------------------------------------------------------------------------------------------ core matrix
@pytest.mark.parametrize("major", MAJORS, ids=MAJOR_IDS)
@pytest.mark.parametrize("shape", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
def test_core_shapes(cuda, shape, major):
    """Every operand-major combination over the edge shapes: smallest, K below one k-block and N below one 32-column
    chunk, exact tiles, ragged everywhere, a ragged last k-block, 48 k-blocks around the stage ring, and more tiles than
    SMs (persistent CTAs carrying stage / phase across tiles, 3 k-blocks not dividing the stage count), and rows whose
    length is not a whole number of 16-byte units (N = 333, 330), which must not write the columns between N and c_ld."""
    M, N, K = shape
    run_gemm(M, N, K, a_mn=major[0], b_mn=major[1], seed_data=M + N + K)
    if N % 8:
        run_gemm(M, N, K, a_mn=major[0], b_mn=major[1], out_dtype=torch.bfloat16, seed_data=M + N + K)


@pytest.mark.parametrize("major", MAJORS, ids=MAJOR_IDS)
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_core_batched(cuda, major, out_dtype):
    """nb1 = 3, nb2 = 2 with distinct padded batch strides on every operand and the output (z = b2 * nb1 + b1)."""
    run_gemm(200, 136, 152, a_mn=major[0], b_mn=major[1], nb1=3, nb2=2, out_dtype=out_dtype, seed_data=5)


@pytest.mark.parametrize("major", MAJORS, ids=MAJOR_IDS)
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_core_broadcast_b(cuda, major, out_dtype):
    """B shared by every batch entry (b_bs = 0): the layout of the relative-position contractions (Q PE^T, dQP PE)."""
    run_gemm(150, 320, 64, a_mn=major[0], b_mn=major[1], nb1=4, nb2=2, b_bcast=(True, True), out_dtype=out_dtype,
             seed_data=6)


# Overlapping windows of the convolutions (rows, K, ld, nb1): row r of a K-major window is the K elements from r * ld.
# Post-net Conv1d k5 (ld = C, K = 5 C), front-end layers 1-4 (ld = 2 C, K = 3 C), the positional conv (ld = cg = 48 / 64,
# K = 128 cg: a row pitch of 96 / 128 bytes, not a multiple of the 128-byte swizzle span for 48), and each family again
# with a ragged last k-block (K % 64 != 0).
KWINDOWS = {"postnet80": (300, 400, 80, 2), "postnet256": (200, 1280, 256, 1), "postnet88_ragged": (130, 440, 88, 2),
            "frontend512": (150, 1536, 1024, 2), "frontend200_ragged": (90, 600, 400, 2),
            "posconv48": (130, 6144, 48, 1), "posconv64": (130, 8192, 64, 1), "posconv48_ragged": (70, 624, 48, 2),
            "posconv64_ragged": (70, 8168, 64, 1)}
# MN-major windows (rows, K, ld, nb1): k-row k is the `rows` elements from k * ld -- the B operand of the weight
# gradients, ld = s C and rows = k C (strided layers, s = 2, k = 3) or ld = C and rows = 5 C (post-net).
MWINDOWS = {"strided64_ragged": (192, 300, 128, 2), "strided512_ragged": (1536, 200, 1024, 1),
            "postnet80": (400, 704, 80, 1), "postnet80_ragged": (400, 700, 80, 2)}
SIDES = [("a", False), ("a", True), ("b", False), ("b", True)]
SIDE_IDS = ["win_a-b_k", "win_a-b_mn", "win_b-a_k", "win_b-a_mn"]


def _run_window(case, mn, side, other_mn, seed):
    rows, K, ld, nb1 = case
    if side == "a":
        run_gemm(rows, 136, K, a_mn=mn, b_mn=other_mn, nb1=nb1, a_win=ld, seed_data=seed)
    else:
        run_gemm(136, rows, K, a_mn=other_mn, b_mn=mn, nb1=nb1, b_win=ld, seed_data=seed)


@pytest.mark.parametrize("side", SIDES, ids=SIDE_IDS)
@pytest.mark.parametrize("case", list(KWINDOWS), ids=list(KWINDOWS))
def test_core_window_k_major(cuda, case, side):
    """A K-major overlapping-window operand (ld < K) against either major of the other operand, on either side."""
    _run_window(KWINDOWS[case], False, side[0], side[1], seed=31)


@pytest.mark.parametrize("side", SIDES, ids=SIDE_IDS)
@pytest.mark.parametrize("case", list(MWINDOWS), ids=list(MWINDOWS))
def test_core_window_mn_major(cuda, case, side):
    """An MN-major overlapping-window operand (ld < rows) against either major of the other operand, on either side."""
    _run_window(MWINDOWS[case], True, side[0], side[1], seed=32)


def test_core_cases_under_both_pinned_tile_widths(cuda):
    """The test_core_* cases again in child processes with ST5_GEMM_BN=64 and =128 (read once per process)."""
    here = os.path.abspath(__file__)
    root = os.path.dirname(os.path.dirname(here))
    for bn in ("64", "128"):
        env = dict(os.environ, ST5_GEMM_BN=bn)
        cp = subprocess.run([sys.executable, "-m", "pytest", here, "-q", "-m", "gpu", "-k", "core and not pinned",
                             "-p", "no:cacheprovider"], cwd=root, env=env, capture_output=True, text=True,
                            timeout=900)
        tail = "\n".join(cp.stdout.splitlines()[-15:])
        assert cp.returncode == 0, f"ST5_GEMM_BN={bn}:\n{tail}\n{cp.stderr[-2000:]}"
        assert " passed" in tail and "skipped" not in tail, tail
        print(f"ST5_GEMM_BN={bn}: {tail.splitlines()[-1]}")


# ------------------------------------------------------------------------------------------------ epilogue matrix
# One mid-size ragged shape per tile width: the cost model (gemm.cu gemm_launch) takes 128 x 64 tiles for 300 x 328
# (9 tiles either way: the narrow tile is cheaper) and 128 x 128 for 1100 x 1496 (108 wide tiles = one round vs 216
# narrow ones = two). The odd-N variants keep c_ld a multiple of 8 (TMA-addressable output).
WIDTHS = {"bn64": (300, 328, 333, 336), "bn128": (1100, 1496, 1499, 1504)}


@pytest.fixture(params=list(WIDTHS), ids=list(WIDTHS))
def width(request):
    return WIDTHS[request.param]


def test_alpha_scales_the_product_only_and_accumulate_1(cuda, width):
    M, N, _, _ = width
    run_gemm(M, N, 200, alpha=0.125, accumulate=1, seed_data=11)
    # alpha on (product + c_old) would move every output by 7/8 |c_old| ~ 0.7: the bound above is ~1e-5


def test_accumulate_2_into_a_shared_output(cuda, width):
    M, N, _, _ = width
    run_gemm(M, N, 96, nb1=3, shared=True, accumulate=2, b_mn=True, a_mn=True, seed_data=12)


@pytest.mark.parametrize("bias", ["aligned", "offset"])
def test_bias(cuda, width, bias):
    """Aligned bias pointer (16-byte vector loads, shuffles only in the ragged last chunk) and a pointer 4 bytes past a
    16-byte boundary (every chunk through the one-load-per-warp + register-shuffle path)."""
    M, N, _, _ = width
    run_gemm(M, N, 200, bias=bias, out_dtype=torch.bfloat16, seed_data=13)
    run_gemm(M, N, 200, bias=bias, seed_data=14)


def test_bias2_rows_and_batches(cuda, width):
    """bias2[m // bias2_rows][n] (row pitch N) on top of bias; the kernel applies the same rows to every batch entry."""
    M, N, _, _ = width
    run_gemm(M, N, 200, bias="aligned", bias2_rows=37, nb1=2, seed_data=15)


@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_residual(cuda, width, out_dtype):
    M, N, _, _ = width
    run_gemm(M, N, 200, residual=True, bias="aligned", out_dtype=out_dtype, seed_data=16)


@pytest.mark.parametrize("act", ["relu", "gelu", "gelu_tanh", "tanh"])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_activation_and_c_pre(cuda, width, act, out_dtype):
    M, N, _, _ = width
    run_gemm(M, N, 200, act=act, c_pre=True, bias="aligned", out_dtype=out_dtype, seed_data=17)


@pytest.mark.parametrize("ag", ["relu", "gelu", "gelu_tanh", "tanh", "gate"])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_actgrad_pre(cuda, width, ag, out_dtype):
    """result *= act'(actgrad_pre[m][n]) (gate: *= actgrad_pre), bf16 through the 16-byte vector path, fp32 per element."""
    M, N, _, _ = width
    run_gemm(M, N, 200, actgrad_act=ag, out_dtype=out_dtype, seed_data=18)


@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("odd", [False, True], ids=["n8", "odd_n"])
def test_dropout_mask_and_scale(cuda, width, p, odd):
    """Kept set == dropout_ref's mask at index (z * M + m) * N + n (N, not c_ld), kept values v / (1 - p). N % 8 == 0
    takes dropout8_apply, odd N (rows starting anywhere in a Philox group) dropout_keep_mask32; nb1 = 2 puts z * M into
    the index."""
    M, N8, Nodd, ld_odd = width
    N, c_ld = (Nodd, ld_odd) if odd else (N8, None)
    r = run_gemm(M, N, 200, act="relu" if p == 0.5 else None, drop_p=p, nb1=2, c_ld=c_ld, out_dtype=torch.float32,
                 seed=0x1234_5678_9ABC, offset=(3 << 32) + 17, seed_data=19)
    keep = r["keep"]
    assert abs(float(keep.double().mean()) - (1 - p)) < 0.01


def test_epilogue_order(cuda, width):
    """dropout(act(alpha v + c_old + bias + bias2)) * act'(pre) + residual, c_pre taken before act, all at once."""
    M, N, _, _ = width
    r = run_gemm(M, N, 200, alpha=0.5, accumulate=1, bias="offset", bias2_rows=50, act="gelu", c_pre=True,
                 drop_p=0.2, actgrad_act="tanh", residual=True, seed_data=20)
    assert torch.isfinite(r["got"]).all()


def test_gelu_tanh_gate_epilogue(cuda, width):
    """fc1 in throughput mode: C = drop(gelu_tanh(x)), c_pre = keep * scale * gelu_tanh'(x), both bf16. The multiplier
    must also equal, bit for bit, what st5_act_bwd's gelu_tanh derivative (the same device function, the same mask at
    the same linear index) gives for the fp32 pre-activation of the same product."""
    from speecht5_b200 import kernels as K_
    M, N, _, _ = width
    p, seed, off = 0.1, 99, 5
    r = run_gemm(M, N, 200, act="gelu_tanh_gate", c_pre=True, drop_p=p, out_dtype=torch.bfloat16, c_ld=N, seed=seed,
                 offset=off, seed_data=21)
    L = r["L"]
    got_pre = L.region(r["got_pre"]).double()
    e = (got_pre - L.region(r["ref_pre"]).double()).abs()
    # gelu_tanh'(x) through the MUFU tanh: |d'/dt| <= 0.5 + |x| (0.8 + 0.11 x^2), |dt| <= 2^-11
    x = r["pre"]
    # (both sides rounded to bf16: one unit in the last place apart at most)
    assert bool((e <= 2.0 ** -7 * got_pre.abs() + 2.0 ** -10 * (1 + x.abs()) ** 3 * D.drop_scale(p) + TINY).all())
    sure = E._gelu_tanh_grad(x).abs() > 1e-3  # (gelu_tanh'(x) itself is 0 in fp32 far left of the origin)
    assert torch.equal((got_pre != 0)[sure], r["keep"][sure]), "gate multiplier: dropped set differs from dropout_ref"
    # cross-check: same product in fp32 (same tile width, same accumulation order), then act_bwd(ones, x32)
    x = run_gemm(M, N, 200, out_dtype=torch.float32, c_ld=N, seed_data=21, check=False)
    x32 = x["got"].float().reshape(-1).contiguous().cuda()
    ones = torch.ones_like(x32)
    d32 = torch.empty_like(x32)
    K_.act_bwd(ones, x32, d32, "gelu_tanh", drop_p=p, seed=seed, offset=off)
    assert torch.equal(d32.to(torch.bfloat16).cpu().double().reshape(got_pre.shape), got_pre)


def test_device_resident_seed(cuda, width):
    """seed = device address of an int64, offset | 1 << 63 (RT.enable_device_seed): the same mask as the host seed."""
    M, N, _, _ = width
    a = run_gemm(M, N, 200, drop_p=0.3, nb1=2, seed=4242, offset=9, seed_data=22)
    b = run_gemm(M, N, 200, drop_p=0.3, nb1=2, seed=4242, offset=9, device_seed=True, seed_data=22)
    assert torch.equal(a["got"], b["got"])


@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_per_thread_store_fallback(cuda, width, out_dtype):
    """Output base one element past a 16-byte boundary: not TMA-addressable, so every row leaves through per-thread
    stores. With bias, residual and odd-N dropout the result must equal the TMA path's bit for bit (same tile width,
    same accumulation order) and stay inside [M) x [N)."""
    M, _, Nodd, ld = width
    kw = dict(bias="aligned", residual=True, drop_p=0.25, nb1=2, c_ld=ld, out_dtype=out_dtype, seed_data=23)
    fb = run_gemm(M, Nodd, 200, misalign=1, **kw)
    tma = run_gemm(M, Nodd, 200, **kw)
    assert torch.equal(fb["got"], tma["got"])


def test_rejected_configurations_do_not_launch(cuda):
    from speecht5_b200 import kernels as K_
    dev = torch.device("cuda")
    a = torch.randn(64, 64, device=dev).to(torch.bfloat16)

    def expect(code, out, **kw):
        before = out.clone()
        with pytest.raises(RuntimeError, match=rf"code {code}\)"):
            K_.gemm(a, a, out, M=64, N=kw.pop("N", 64), K=64, **kw)
        torch.cuda.synchronize()
        assert torch.equal(out.isnan(), before.isnan()) and torch.equal(out.nan_to_num(), before.nan_to_num())

    bf = torch.full((64 * 64,), NAN, device=dev, dtype=torch.bfloat16)
    f32 = torch.full((64 * 64 + 64,), NAN, device=dev)
    expect(-3, bf, accumulate=1)                                           # accumulate into bf16
    expect(-5, bf, N=63, c_ld=64, act="gelu_tanh_gate", c_pre=bf.clone())  # gate, odd N
    expect(-5, f32, act="gelu_tanh_gate", c_pre=f32.clone())              # gate, fp32 output
    expect(-6, f32, N=63, c_ld=63, accumulate=2)                           # L2 reduce, rows not 16-byte aligned
    expect(-6, f32, N=62, c_ld=64, accumulate=2)                           # L2 reduce, ragged row length
    expect(-7, f32, nb1=2, a_bs=(0, 0), b_bs=(0, 0), c_bs=(0, 0))          # shared output without accumulate = 2
