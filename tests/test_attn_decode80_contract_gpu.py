"""-m gpu: the head-dimension entry points of the one-row attention (st5_attn_decode_hd_fwd, st5_attn_lineage_hd_fwd) and
the wide LayerNorm forward (st5_ln_fwd_wide) called through ctypes against fp64 statements with ELEMENTWISE bounds, on
buffers laid out with NaN sentinels everywhere the contract does not let a kernel read or write:
  - q / k / v live in fused q|k|v rows whose other column blocks are NaN; the K / V rows of masked keys and the rows
    [Tk, buffer) are NaN; out rows have a NaN gap past H * 80; every buffer has NaN guard zones; scratch starts NaN;
  - lineage: the rows a query row does not read (other lineages) are NaN at the positions it does not own.
Head dim 80 over Tk below, at and across 64 (splits), bf16 and fp32, masks, kv_div and lineage tables; each row
bit-identical across B and key span; head dim 64 through the new entry points bit-identical to st5_attn_decode_fwd /
st5_attn_lineage_fwd; rejected configurations write nothing. LayerNorm at C in {1032, 1280, 2048} with and without a
residual; C = 1032 still rejected by st5_ln_fwd."""
import ctypes as ct
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

NAN = float("nan")
G = 64
F32, BF16, F64 = torch.float32, torch.bfloat16, torch.float64
DT = {F32: 0, BF16: 1}
U = {F32: 2.0 ** -24, BF16: 2.0 ** -8}
DCH = 64
REPORT = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if REPORT:
        print("\nlargest err / bound per entry point:")
        for k in sorted(REPORT):
            print(f"  {k:44s} {REPORT[k]:.3g}")


def _lib():
    from speecht5_b200 import _lib as L
    return L.load()


def _st():
    return ct.c_void_p(torch.cuda.current_stream().cuda_stream)


class Buf:
    def __init__(self, n, dtype=F32, fill=None):
        self.flat = torch.full((2 * G + n,), NAN, dtype=dtype, device="cuda")
        self.t = self.flat[G:G + n]
        if fill is not None:
            self.t.copy_(torch.as_tensor(fill).reshape(-1).to(dtype))

    def untouched(self, what):
        g = torch.cat([self.flat[:G], self.flat[G + self.t.numel():]]).float()
        assert bool(torch.isnan(g).all()), f"{what}: guard zone written"

    def snapshot(self):
        return self.flat.clone()

    def same_as(self, snap):
        w = torch.int16 if self.flat.dtype == BF16 else torch.int32
        return bool(torch.equal(self.flat.view(w), snap.view(w)))


def _check(name, got, ref, bound):
    err = (got.double() - ref).abs()
    ratio = torch.where(torch.isfinite(got.double()), err / bound, torch.full_like(err, math.inf))
    worst = float(ratio.max()) if ratio.numel() else 0.0
    REPORT[name] = max(REPORT.get(name, 0.0), worst)
    assert worst <= 1.0, f"{name}: max err / bound {worst:.3g}"


# ====================================================================================== one-row attention, any head dim
def _inputs(Bkv, H, Tk, hd, dtype, seed, nq=None):
    g = torch.Generator().manual_seed(seed)
    sig = math.sqrt(3.0)
    q = (torch.randn(nq or Bkv, H, hd, generator=g) * sig / hd ** 0.25).to(dtype)
    k = (torch.randn(Bkv, H, Tk, hd, generator=g) * sig / hd ** 0.25).to(dtype)
    v = torch.randn(Bkv, H, Tk, hd, generator=g).to(dtype)
    return q, k, v


def reference(q, k, v, scale, key_pad, rows):
    """fp64 softmax attention of query row b over keys k[rows[b, j], :, j] (rows [Bq, Tk] long); a row with every key
    masked gives zeros. Returns out [Bq, H, hd], P [Bq, H, Tk] and the bound inputs."""
    Bq, Tk = rows.shape
    j = torch.arange(Tk)[None].expand(Bq, Tk)
    kg = k.double().permute(0, 2, 1, 3)[rows, j]          # [Bq, Tk, H, hd]
    vg = v.double().permute(0, 2, 1, 3)[rows, j]
    qd = q.double()
    s = torch.einsum("bhc,bjhc->bhj", qd, kg) * scale
    smag = torch.einsum("bhc,bjhc->bhj", qd.abs(), kg.abs()) * scale
    ok = torch.ones_like(s, dtype=torch.bool) if key_pad is None else ~key_pad.bool()[:, None, :].expand_as(s)
    s = s.masked_fill(~ok, -math.inf)
    P = torch.nan_to_num(torch.softmax(s, -1), nan=0.0)
    out = torch.einsum("bhj,bjhc->bhc", P, vg)
    return dict(out=out, P=P, smag=torch.where(ok, smag, 0.0), s=torch.where(ok, s, 0.0), vabs=vg.abs())


def bounds(f, ns, u):
    """Elementwise bounds. Score of a key: 8 sequential fp32 products per thread, then ten thread partials added in
    order (depth <= 18, Cs = 80 units of 2^-24 on |q|.|k| + |s| + the row's largest + 4, as tests/attention_ref.py
    states for the 64-wide kernel); the denominator: a 5-level shuffle tree, 4 warp partials and ns merges; each output
    channel: <= 6 sequential keys per thread, 12 slot partials in order and ns merges."""
    es = 80 * 2.0 ** -24 * (f["smag"] + f["s"].abs() + (f["smag"] + f["s"].abs()).amax(-1, keepdim=True) + 4.0)
    el = es.amax(-1, keepdim=True) + (ns + 16) * 2.0 ** -24
    EP = f["P"] * (es + el + 2 * 2.0 ** -24)
    b_out = (ns + 32) * 2.0 ** -24 * torch.einsum("bhj,bjhc->bhc", f["P"], f["vabs"]) \
        + torch.einsum("bhj,bjhc->bhc", EP, f["vabs"]) + u * f["out"].abs() + 1e-30
    return b_out, EP + 1e-30


class Layout:
    """k / v of Bkv batch rows in fused q|k|v rows of width 3 H hd + 8 (other blocks NaN), Tbuf >= Tk rows each, key
    rows no query row reads NaN; Bq query rows in rows of the same width; out rows of pitch H hd + 32 (gaps NaN)."""

    def __init__(self, q, k, v, hd, dtype, rows, key_pad, Tbuf=None, probs=True, ws=True):
        Bq, H = q.shape[0], q.shape[1]
        Bkv, Tk = k.shape[0], k.shape[2]
        self.Bq, self.H, self.Tk, self.hd, self.dtype = Bq, H, Tk, hd, dtype
        Tbuf = Tbuf or Tk + 3
        W = 3 * H * hd + 8
        qh = torch.full((Bq, W), NAN)
        qh[:, :H * hd] = q.reshape(Bq, H * hd).float()
        read = torch.zeros(Bkv, Tk, dtype=torch.bool)
        for b in range(Bq):
            for j in range(Tk):
                if key_pad is None or key_pad[b, j] == 0:
                    read[rows[b, j], j] = True
        kv = torch.full((Bkv, Tbuf, W), NAN)
        kv[:, :Tk, H * hd:2 * H * hd] = k.transpose(1, 2).reshape(Bkv, Tk, H * hd).float()
        kv[:, :Tk, 2 * H * hd:3 * H * hd] = v.transpose(1, 2).reshape(Bkv, Tk, H * hd).float()
        kv[:, :Tk][~read] = NAN
        self.qb, self.kvb = Buf(qh.numel(), dtype, qh), Buf(kv.numel(), dtype, kv)
        self.o_bs = H * hd + 32
        self.out = Buf(Bq * self.o_bs, dtype)
        self.probs = Buf(Bq * H * Tk) if probs else None
        nws = _lib().st5_attn_decode_hd_ws_floats(Bq, H, Tk, int(probs), hd)
        self.ws = Buf(nws) if ws and nws > 0 else None
        self.kp = key_pad.cuda().contiguous() if key_pad is not None else None
        self.W, self.Tbuf = W, Tbuf

    def args(self, scale, k_off=0):
        from speecht5_b200 import _lib as L
        H, hd = self.H, self.hd
        a = L.AttnDecodeArgs()
        a.B, a.H, a.Tk, a.dtype = self.Bq, H, self.Tk, DT[self.dtype]
        esz = 4 if self.dtype == F32 else 2
        base = self.kvb.t.data_ptr()
        a.q, a.q_bs = self.qb.t.data_ptr(), self.W
        a.k, a.k_ld, a.k_bs = base + (H * hd + k_off) * esz, self.W, self.Tbuf * self.W
        a.v, a.v_ld, a.v_bs = base + 2 * H * hd * esz, self.W, self.Tbuf * self.W
        a.key_pad = self.kp.data_ptr() if self.kp is not None else None
        a.out, a.o_bs = self.out.t.data_ptr(), self.o_bs
        a.probs = self.probs.t.data_ptr() if self.probs is not None else None
        a.scale = scale
        a.ws = self.ws.t.data_ptr() if self.ws is not None else None
        return a

    def run(self, scale, head_dim=None, lineage=None, old=False, k_off=0):
        lib = _lib()
        a = self.args(scale, k_off)
        if lineage is None:
            rc = lib.st5_attn_decode_fwd(ct.byref(a), _st()) if old else \
                lib.st5_attn_decode_hd_fwd(ct.byref(a), self.hd if head_dim is None else head_dim, _st())
        else:
            from speecht5_b200 import _lib as L
            la = L.AttnLineageArgs()
            la.base = a
            tab, div = lineage
            la.kv_rows, la.kv_rows_ld, la.kv_div = (tab.data_ptr() if tab is not None else None,
                                                    tab.stride(0) if tab is not None else 0, div)
            rc = lib.st5_attn_lineage_fwd(ct.byref(la), _st()) if old else \
                lib.st5_attn_lineage_hd_fwd(ct.byref(la), self.hd if head_dim is None else head_dim, _st())
        torch.cuda.synchronize()
        return rc

    def bufs(self):
        return [b for b in (self.qb, self.kvb, self.out, self.probs, self.ws) if b is not None]

    def out_rows(self):
        o = self.out.t.view(self.Bq, self.o_bs)
        assert bool(torch.isnan(o[:, self.H * self.hd:].float()).all()), "out: gap between rows written"
        return o[:, :self.H * self.hd].reshape(self.Bq, self.H, self.hd)


def _ragged(B, Tk, seed):
    g = torch.Generator().manual_seed(seed)
    L = [Tk] + [int(torch.randint(1, Tk + 1, (1,), generator=g)) for _ in range(B - 1)]
    return (torch.arange(Tk)[None, :] >= torch.tensor(L)[:, None]).to(torch.uint8)


def _run_and_check(name, q, k, v, hd, dtype, rows, key_pad, scale, probs=True, lineage=None, Tbuf=None):
    lay = Layout(q, k, v, hd, dtype, rows, key_pad, Tbuf=Tbuf, probs=probs and lineage is None)
    assert lay.run(scale, lineage=lineage) == 0, _lib().st5_last_error()
    f = reference(q, k, v, scale, key_pad, rows)
    ns = -(-k.shape[2] // DCH)
    b_out, b_p = bounds(f, ns, U[dtype])
    for buf in lay.bufs():
        buf.untouched(name)
    out = lay.out_rows()
    _check(f"{name} out", out.cpu(), f["out"], b_out)
    if lay.probs is not None:
        _check(f"{name} probs", lay.probs.t.view(lay.Bq, lay.H, lay.Tk).cpu(), f["P"], b_p)
    return lay, out.clone()


@pytest.mark.parametrize("i,Tk", list(enumerate([1, 40, 63, 64, 65, 128, 129, 300, 1500])))
@pytest.mark.parametrize("dtype", [F32, BF16])
def test_decode80(cuda, i, Tk, dtype):
    B, H = [(1, 1), (3, 16), (8, 2)][i % 3]
    q, k, v = _inputs(B, H, Tk, 80, dtype, seed=200 + i)
    key_pad = None if i % 2 == 0 else _ragged(B, Tk, i)
    rows = torch.arange(B)[:, None].expand(B, Tk)
    _run_and_check(f"decode80 {dtype}", q, k, v, 80, dtype, rows, key_pad, 80 ** -0.5, probs=i % 4 != 3)


@pytest.mark.parametrize("Tk", [17, 64, 100, 257])
@pytest.mark.parametrize("dtype", [F32, BF16])
def test_lineage80_table_and_div(cuda, Tk, dtype):
    """A lineage table (each key from another batch row, as beam search reorders) with a causal-style pad, and kv_div
    (query rows sharing one utterance's keys)."""
    Bkv, H = 6, 4
    g = torch.Generator().manual_seed(Tk)
    q, k, v = _inputs(Bkv, H, Tk, 80, dtype, seed=300 + Tk)
    tab = torch.randint(0, Bkv, (Bkv, Tk + 5), generator=g, dtype=torch.int32)
    kp = (torch.arange(Tk)[None] > torch.randint(0, Tk, (Bkv, 1), generator=g)).to(torch.uint8)
    _run_and_check(f"lineage80 rows {dtype}", q, k, v, 80, dtype, tab[:, :Tk].long(), kp, 80 ** -0.5,
                   lineage=(tab.cuda(), 1))
    div = 3
    q2, _, _ = _inputs(Bkv, H, Tk, 80, dtype, seed=400 + Tk, nq=Bkv * div)
    rows = (torch.arange(Bkv * div) // div)[:, None].expand(Bkv * div, Tk)
    kp2 = (torch.arange(Tk)[None] > torch.randint(0, Tk, (Bkv * div, 1), generator=g)).to(torch.uint8)
    _run_and_check(f"lineage80 div {dtype}", q2, k, v, 80, dtype, rows, kp2, 80 ** -0.5, lineage=(None, div))


@pytest.mark.parametrize("dtype", [F32, BF16])
def test_decode80_rows_are_bit_identical_across_batch_and_span(cuda, dtype):
    """Edge masks (a single key, a dead split between valid ones, every key masked -> zeros) in a batch of 5, then each
    row alone and inside a wider key span: outputs and probabilities bit for bit."""
    B, H, Tk = 5, 3, 200
    q, k, v = _inputs(B, H, Tk, 80, dtype, seed=11)
    kp = torch.zeros(B, Tk, dtype=torch.uint8)
    kp[0, 1:] = 1
    kp[1, 64:128] = 1
    kp[2, :] = 1
    kp[3, 77:] = 1
    rows = torch.arange(B)[:, None].expand(B, Tk)
    lay, out = _run_and_check(f"decode80 {dtype}", q, k, v, 80, dtype, rows, kp, 0.11)
    pr = lay.probs.t.view(B, H, Tk).clone()
    assert bool((out[2] == 0).all()) and bool((pr[2] == 0).all())
    w = torch.int32 if dtype == F32 else torch.int16
    extra = 150
    g = torch.Generator().manual_seed(12)
    k2 = torch.cat([k, torch.randn(B, H, extra, 80, generator=g).to(dtype)], 2)
    v2 = torch.cat([v, torch.randn(B, H, extra, 80, generator=g).to(dtype)], 2)
    kp2 = torch.cat([kp, torch.ones(B, extra, dtype=torch.uint8)], 1)
    wide = Layout(q, k2, v2, 80, dtype, torch.arange(B)[:, None].expand(B, Tk + extra), kp2)
    assert wide.run(0.11) == 0
    assert torch.equal(wide.out_rows().contiguous().view(w), out.contiguous().view(w))
    p2 = wide.probs.t.view(B, H, Tk + extra)
    assert torch.equal(p2[..., :Tk].contiguous().view(torch.int32), pr.contiguous().view(torch.int32))
    for b in (0, 1, 3, 4):
        one = Layout(q[b:b + 1], k[b:b + 1], v[b:b + 1], 80, dtype, torch.zeros(1, Tk, dtype=torch.long), kp[b:b + 1])
        assert one.run(0.11) == 0
        assert torch.equal(one.out_rows()[0].contiguous().view(w), out[b].contiguous().view(w)), b
    # Tk <= 64 (one split, written directly) against the same keys inside a two-split span
    s1 = Layout(q, k[:, :, :50], v[:, :, :50], 80, dtype, rows[:, :50], kp[:, :50])
    assert s1.run(0.11) == 0
    kp3 = torch.cat([kp[:, :50], torch.ones(B, 30, dtype=torch.uint8)], 1)
    s2 = Layout(q, k[:, :, :80], v[:, :, :80], 80, dtype, rows[:, :80], kp3)
    assert s2.run(0.11) == 0
    assert torch.equal(s1.out_rows().contiguous().view(w), s2.out_rows().contiguous().view(w))


@pytest.mark.parametrize("Tk", [30, 64, 200])
@pytest.mark.parametrize("dtype", [F32, BF16])
def test_head_dim_64_through_the_new_entry_points_is_the_old_kernel(cuda, Tk, dtype):
    B, H = 4, 12
    q, k, v = _inputs(B, H, Tk, 64, dtype, seed=500 + Tk)
    kp = _ragged(B, Tk, Tk)
    rows = torch.arange(B)[:, None].expand(B, Tk)
    w = torch.int32 if dtype == F32 else torch.int16
    for lineage in (None, (None, 1)):
        a, b = (Layout(q, k, v, 64, dtype, rows, kp, probs=lineage is None) for _ in range(2))
        assert a.run(0.125, lineage=lineage, old=True) == 0 and b.run(0.125, lineage=lineage) == 0
        assert torch.equal(a.out.flat.view(w), b.out.flat.view(w))
        if a.probs is not None:
            assert torch.equal(a.probs.flat.view(torch.int32), b.probs.flat.view(torch.int32))
    assert _lib().st5_attn_decode_hd_ws_floats(B, H, Tk, 1, 64) == _lib().st5_attn_decode_ws_floats(B, H, Tk, 1)


@pytest.mark.parametrize("dtype", [F32, BF16])
@pytest.mark.parametrize("what,want", [("head_dim", -2), ("ws", -5), ("k", -6), ("div", -2)])
def test_decode80_rejections_write_nothing(cuda, dtype, what, want):
    B, H, Tk = 2, 2, 100
    q, k, v = _inputs(B, H, Tk, 80, dtype, seed=13)
    rows = torch.arange(B)[:, None].expand(B, Tk)
    lay = Layout(q, k, v, 80, dtype, rows, _ragged(B, Tk, 3), probs=False)
    if what == "ws":
        lay.ws = None
    snaps = [b.snapshot() for b in lay.bufs()]
    kw = dict(head_dim=dict(head_dim=96), k=dict(k_off=1), div=dict(lineage=(None, 0))).get(what, {})
    assert lay.run(0.125, **kw) == want
    assert all(b.same_as(s) for b, s in zip(lay.bufs(), snaps))
    assert _lib().st5_attn_decode_hd_ws_floats(B, H, Tk, 0, 32) == -2


# ================================================================================================= wide LayerNorm
@pytest.mark.parametrize("C", [1032, 1280, 2048])
@pytest.mark.parametrize("dtype", [F32, BF16])
@pytest.mark.parametrize("res", [False, True])
def test_ln_fwd_wide(cuda, C, dtype, res):
    rows = 37
    g = torch.Generator().manual_seed(C + res)
    x = (torch.randn(rows, C, generator=g) * 2 + 0.5).to(dtype)
    r = (torch.randn(rows, C, generator=g)).to(dtype) if res else None
    gamma, beta = torch.randn(C, generator=g), torch.randn(C, generator=g)
    bx, br = Buf(rows * C, dtype, x), (Buf(rows * C, dtype, r) if res else None)
    bg, bb = Buf(C, F32, gamma), Buf(C, F32, beta)
    by, bm, bs = Buf(rows * C, dtype), Buf(rows), Buf(rows)
    rc = _lib().st5_ln_fwd_wide(ct.c_void_p(bx.t.data_ptr()), ct.c_void_p(br.t.data_ptr()) if res else None,
                                ct.c_void_p(bg.t.data_ptr()), ct.c_void_p(bb.t.data_ptr()), ct.c_void_p(by.t.data_ptr()),
                                ct.c_void_p(bm.t.data_ptr()), ct.c_void_p(bs.t.data_ptr()), DT[dtype], rows, C, 1e-5,
                                _st())
    torch.cuda.synchronize()
    assert rc == 0
    for b in (bx, by, bm, bs, bg, bb):
        b.untouched("ln_fwd_wide")
    s = x.double() + (r.double() if res else 0.0)
    mu = s.mean(-1, keepdim=True)
    var = s.var(-1, unbiased=False, keepdim=True)
    rs = 1 / torch.sqrt(var + 1e-5)
    xh = (s - mu) * rs
    y = xh * gamma.double() + beta.double()
    # fp32 statistics over C terms (sequential within a lane, 5 shuffle levels): mean and variance to (C/32 + 8) 2^-24
    # relative to their magnitudes; y inherits |xh| |gamma| times that, plus its own storage rounding
    e = (C / 32 + 16) * 2.0 ** -24 * (1 + (s.abs().mean(-1, keepdim=True) + s.abs().amax(-1, keepdim=True)) * rs)
    bound = e * (xh.abs() + 1) * gamma.double().abs() + U[dtype] * y.abs() + 4 * 2.0 ** -24 * (beta.double().abs() + 1)
    _check(f"ln_fwd_wide {dtype}", by.t.view(rows, C).cpu(), y, bound)
    _check("ln_fwd_wide mean", bm.t.cpu(), mu[:, 0], (C / 32 + 8) * 2.0 ** -24 * s.abs().mean(-1) + 1e-30)
    _check("ln_fwd_wide rstd", bs.t.cpu(), rs[:, 0], e[:, 0] * rs[:, 0] * 2)


@pytest.mark.parametrize("C", [4, 12, 2056, 4096])
def test_ln_rejections_write_nothing(cuda, C):
    rows = 3
    bx, by = Buf(rows * C), Buf(rows * C)
    bg = Buf(C, F32, torch.ones(C))
    snaps = [b.snapshot() for b in (bx, by)]
    P = lambda b: ct.c_void_p(b.t.data_ptr())  # noqa: E731
    assert _lib().st5_ln_fwd_wide(P(bx), None, P(bg), P(bg), P(by), None, None, 0, rows, C, 1e-5, _st()) == -2
    assert bx.same_as(snaps[0]) and by.same_as(snaps[1])
    # st5_ln_fwd keeps its 1024 limit
    b2, y2 = Buf(rows * 1032, F32, torch.randn(rows * 1032, generator=torch.Generator().manual_seed(C))), Buf(rows * 1032)
    g2 = Buf(1032, F32, torch.ones(1032))
    assert _lib().st5_ln_fwd(P(b2), None, P(g2), P(g2), P(y2), None, None, None, 0, rows, 1032, 1e-5, 0.0, 0, 0,
                             _st()) == -2
