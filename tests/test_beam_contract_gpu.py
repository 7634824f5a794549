"""-m gpu: the beam-search entry points of include/speecht5_b200.h (st5_beam_topk, st5_beam_update,
st5_attn_lineage_fwd) called through ctypes, against fp64 statements with elementwise bounds, on buffers with NaN
sentinels wherever the contract does not let a kernel read or write:
  - st5_beam_topk on a grid of dtypes, K, V (2, 3, 2K - 1, 2K, 2K + 1, 81, 8000, 32768), row pitches ld > V with NaN
    padding, temperatures and steps (t = 0, t < min_len, t >= max_len, both, ordinary), with an all -inf row, an all
    -inf sentence, NaN and +inf rows, -inf on eos and rows tied across beams; every sentence's list goes through the
    rank checker of tests/beam_contract_ref.py. ws and the candidate buffers start NaN; entries >= n stay NaN.
  - st5_beam_topk and st5_beam_update in lockstep over whole searches past steps 64 and 128, on logits that are a
    function of each row's token prefix (rebuilt every step from the device's lineage table), against
    tests/beam_ref.update applied to the device's own state and candidates: every state tensor equal every step.
  - st5_attn_lineage_fwd over lineage tables of a search history, with every cache cell the table does not name NaN,
    against tests/attention_ref.decode_forward on explicitly gathered keys, probabilities included; bit-identical
    across B, key spans and kv_div = K against a repeat_interleaved cache.
  - every negative return leaves every buffer bit-identical.
The largest err / bound per entry point and the largest step the searches reached are printed at the end (-s)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import attention_ref as A
import beam_contract_ref as BR
import beam_ref
import rowops_ref
from test_attention_contract_gpu import Flat
from test_beam_gpu import _random_history, _state

pytestmark = pytest.mark.gpu

NAN, INF = float("nan"), float("inf")
F32, BF16 = torch.float32, torch.bfloat16
DT = {F32: 0, BF16: 1}
REPORT = {}
STEPS = {}


@pytest.fixture(autouse=True)
def _device(cuda):
    yield


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if REPORT:
        print("\nlargest err / bound per entry point:")
        for k in sorted(REPORT):
            print(f"  {k:40s} {REPORT[k]:.3g}")
    if STEPS:
        print(f"largest step t reached by the lockstep searches: {max(STEPS.values())}")


def _lib():
    from speecht5_b200 import _lib as L
    return L.load()


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def P(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _ints(f):
    """An int32 view of a fp32 Flat: NaN bits (0x7fc00000) are the sentinel."""
    return f.t.view(torch.int32)


def _bits(t):
    return t.contiguous().view(torch.int16 if t.dtype in (BF16, torch.float16) else
                               torch.int32 if t.element_size() == 4 else torch.int64 if t.element_size() == 8
                               else torch.uint8)


def _scalars(*v):
    return [torch.tensor([x], dtype=torch.int64, device="cuda") for x in v]


def _beam_n(t, K, V):
    return min(2 * K, (V if t == 0 else K * V) - 1)


# ============================================================================================ st5_beam_topk
class TopK:
    """Logits [BK, ld] (columns >= V NaN), cum, mask, ws and cand_* [B, 2K], all inside NaN buffers with guards."""

    def __init__(self, x, cum, mask, K, ld_pad):
        BK, V = x.shape
        self.B, self.K, self.V, self.ld = BK // K, K, V, V + ld_pad
        self.dtype = x.dtype
        self.lg = Flat((BK, self.ld), x.dtype)
        self.lg.t[:, :V] = x.cuda()
        self.cum, self.mask = Flat((BK,), F32), Flat((V,), F32)
        self.cum.t.copy_(cum)
        self.mask.t.copy_(mask)
        self.ws = Flat((max(1, _lib().st5_beam_topk_ws_floats(self.B, K)),), F32)
        self.cs, self.ct, self.cb = (Flat((self.B, 2 * K), F32) for _ in range(3))

    def bufs(self):
        return [self.lg, self.cum, self.mask, self.ws, self.cs, self.ct, self.cb]

    def run(self, inv_temp, eos, tt, mnt, mxt, **over):
        a = dict(logits=P(self.lg.t), ld=self.ld, dtype=DT[self.dtype], B=self.B, K=self.K, V=self.V,
                 cum=P(self.cum.t), mask=P(self.mask.t), inv_temp=float(inv_temp), eos=eos, t=P(tt), mn=P(mnt),
                 mx=P(mxt),
                 cs=P(self.cs.t), ct=P(self.ct.t), cb=P(self.cb.t), ws=P(self.ws.t))
        a.update(over)
        rc = _lib().st5_beam_topk(*a.values(), _st())
        torch.cuda.synchronize()
        return rc


def _check_topk(name, x, cum, mask, inv_temp, eos, t, mn, mx, K, tk):
    B, V = tk.B, tk.V
    n = _beam_n(t, K, V)
    for b in (tk.lg, tk.cum, tk.mask, tk.ws, tk.cs, tk.ct, tk.cb):
        b.untouched(name)
    cs, ct, cb = tk.cs.t.cpu(), _ints(tk.ct).cpu(), _ints(tk.cb).cpu()
    nan_bits = int(torch.tensor([NAN]).view(torch.int32))
    assert bool(torch.isnan(cs[:, n:]).all()) and bool((ct[:, n:] == nan_bits).all()) and \
        bool((cb[:, n:] == nan_bits).all()), f"{name}: entries >= n written"
    z, bnd = BR.scores(x, cum, mask, inv_temp, eos, t, mn, mx, K)
    for s in range(B):
        same = BR.same_inputs(x, cum, mask, eos, K, s, t)
        w = BR.check_sentence(z[s], bnd[s], cs[s, :n], ct[s, :n], cb[s, :n], V, same, what=f"{name} sentence {s}")
        key = f"beam_topk {'bf16' if x.dtype == BF16 else 'f32'}"
        REPORT[key] = max(REPORT.get(key, 0.0), w)
    return cs[:, :n], ct[:, :n], cb[:, :n]


def _topk_inputs(B, K, V, dtype, g):
    """Even rows on a 1/8 grid (exact ties inside a row), odd rows N(0, 9); sentence 0 has rows 0 and K - 1 identical
    (logits and cum: ties across beams); sentence 1: a NaN in beam 0, beam K - 1 all -inf; sentence 2: +inf in beam
    min(1, K - 1); the last sentence (B >= 4) all -inf."""
    BK = B * K
    x = torch.randn(BK, V, generator=g) * 3
    x[0::2] = torch.randint(-32, 33, (len(range(0, BK, 2)), V), generator=g).float() / 8
    x[:, min(3, V - 1)] = torch.where(torch.arange(BK) % 3 == 0, -INF, x[:, min(3, V - 1)])
    cum = -torch.rand(BK, generator=g) * 4
    x[K - 1], cum[K - 1] = x[0], cum[0]
    if B >= 2:
        x[K, V // 2] = NAN
        if K > 1:
            x[2 * K - 1] = -INF
    if B >= 3:
        x[2 * K + min(1, K - 1), V - 1] = INF
    if B >= 4:
        x[(B - 1) * K:] = -INF
    return x.to(dtype), cum


def _grid():
    out = []
    for K in (1, 2, 5, 15, 16):
        for V in sorted({2, 3, 2 * K - 1, 2 * K, 2 * K + 1, 81, 8000, 32768}):
            if V < 2:
                continue
            out.append((K, V))
    return out


GRID = _grid()
STEP_KINDS = ((0, 1, 20), (3, 5, 20), (20, 1, 20), (7, 10, 5), (5, 1, 20))  # t=0, t<min, t>=max, both, ordinary


@pytest.mark.parametrize("i,K,V", [(i, K, V) for i, (K, V) in enumerate(GRID)])
@pytest.mark.parametrize("dtype", [F32, BF16])
def test_topk_grid(i, K, V, dtype):
    B = 64 if (K == 16 and V == 81) else 2 if V >= 8000 and K >= 15 else 4 if V >= 8000 else 5
    g = torch.Generator().manual_seed(1000 * K + V + (7 if dtype == BF16 else 0))
    x, cum = _topk_inputs(B, K, V, dtype, g)
    eos = min(2, V - 1)
    inv_temp = (0.5, 1.0, 1.25)[i % 3]
    ld_pad = 8 * ((i + (dtype == BF16)) % 2)
    for si, (t, mn, mx) in enumerate(STEP_KINDS):
        mask = torch.zeros(V)
        if V > 4:
            mask[V - 1], mask[1] = -0.5, -INF
        if si == 4 and i % 2 == 0:
            mask[eos] = -INF
        tk = TopK(x, cum, mask, K, ld_pad)
        tt, mnt, mxt = _scalars(t, mn, mx)
        assert tk.run(inv_temp, eos, tt, mnt, mxt) == 0
        name = f"topk K={K} V={V} {dtype} t={t} min={mn} max={mx} ld={tk.ld}"
        cs, ct, cb = _check_topk(name, x, cum, mask, inv_temp, eos, t, mn, mx, K, tk)
        if B >= 4:
            assert bool((cs[B - 1] == -INF).all())
            assert (cb[B - 1] * V + ct[B - 1]).tolist() == list(range(cs.shape[1]))
        if si == 3:
            assert bool((cs == -INF).all())


def test_topk_workspace_rows_beyond_beam0_unread_at_t0():
    """At t = 0 only beam 0 takes part: NaN and +inf in the other beams change nothing, and their ws rows stay NaN."""
    K, V, B = 4, 81, 3
    g = torch.Generator().manual_seed(3)
    x, cum = _topk_inputs(B, K, V, F32, g)
    x[1::K] = NAN
    x[2::K, 0] = INF
    tk = TopK(x, cum, torch.zeros(V), K, 8)
    tt, mnt, mxt = _scalars(0, 1, 20)
    assert tk.run(1.0, 2, tt, mnt, mxt) == 0
    _check_topk("topk t=0 other beams", x, cum, torch.zeros(V), 1.0, 2, 0, 1, 20, K, tk)
    ws = tk.ws.t.view(B * K, -1).cpu()
    assert bool(torch.isnan(ws[[r for r in range(B * K) if r % K]]).all())


TOPK_REJECT = [("K0", -2), ("K17", -2), ("V1", -2), ("V32769", -2), ("eos-1", -2), ("eosV", -2), ("B0", -2),
               ("ld", -6)] + [(f"null:{p}", -3) for p in ("logits", "cum", "mask", "t", "mn", "mx", "cs", "ct", "cb",
                                                           "ws")]


@pytest.mark.parametrize("what,want", TOPK_REJECT)
def test_topk_rejections_leave_buffers_untouched(what, want):
    K, V, B = 4, 81, 2
    g = torch.Generator().manual_seed(4)
    x, cum = _topk_inputs(B, K, V, BF16, g)
    tk = TopK(x, cum, torch.zeros(V), K, 8)
    tt, mnt, mxt = _scalars(3, 1, 20)
    snaps = [b.flat.clone() for b in tk.bufs()]
    over = {"K0": dict(K=0), "K17": dict(K=17), "V1": dict(V=1), "V32769": dict(V=32769, ld=32769),
            "eos-1": dict(eos=-1), "eosV": dict(eos=V), "B0": dict(B=0), "ld": dict(ld=V - 1)}.get(what, {})
    if what.startswith("null:"):
        over = {what[5:]: None}
    eos = over.pop("eos", 2)
    assert tk.run(1.0, eos, tt, mnt, mxt, **over) == want
    assert all(torch.equal(_bits(b.flat), _bits(s)) for b, s in zip(tk.bufs(), snaps)), what


# ============================================================================================ lockstep searches
M31 = (1 << 31) - 1


def _mix(h):
    """A 31-bit integer hash, elementwise on non-negative int64 < 2^31 (no product exceeds 2^62)."""
    for c in (0x2C1B3C6D, 0x297A2D39, 0x1B873593):
        h = (h ^ (h >> 15)) & M31
        h = (h * c) & M31
    return h ^ (h >> 13)


class Prefix:
    """Logits of every row as a function of its own token prefix tok[lin[r][j]][j], j = 1..t, rebuilt each step from the
    device's table; eos is weak (-6) before the sentence's step E_s and then drawn around +3 (strong in some rows)."""

    def __init__(self, B, K, V, eos, E, T, dtype, seed):
        self.B, self.K, self.V, self.eos, self.E, self.dtype = B, K, V, eos, E, dtype
        g = torch.Generator().manual_seed(seed)
        self.w = torch.randint(1, 1 << 20, (T,), generator=g, dtype=torch.int64)
        self.salt = (torch.arange(V, dtype=torch.int64) * 0x9E3779B1) & M31

    def __call__(self, lin, tok, t):
        BK = lin.shape[0]
        j = torch.arange(1, t + 1)
        pref = tok[lin[:, 1:t + 1].long(), j].long() if t > 0 else torch.zeros(BK, 0, dtype=torch.int64)
        h = ((pref + 1) * self.w[1:t + 1]).sum(1) + t * 7919
        h = _mix(h & M31)
        u = _mix((h[:, None] ^ self.salt[None]) & M31).double() / 2.0 ** 31
        x = (u * 128).floor() / 16 - 4                       # [-4, 4) on a 1/16 grid
        s = torch.arange(BK) // self.K
        strong = torch.tensor([t >= e for e in self.E])[s]
        x[:, self.eos] = torch.where(strong, 1.0 + 4 * u[:, self.eos], torch.full_like(u[:, self.eos], -6.0))
        return x.to(self.dtype)


NAMES = ("t", "max_len", "cand_score", "cand_token", "cand_beam", "lin", "tok", "score", "ignore", "finished", "parent",
         "cur_tok", "cur_score", "fin_n", "fin_tok", "fin_pos", "fin_len", "fin_score", "stop")


def _update(st, B, K, V, T, eos, normalize, len_penalty, over=None):
    p = {n: P(st[n]) for n in NAMES}
    a = dict(B=B, K=K, V=V, T=T, eos=eos)
    a.update(over or {})
    for n in list(a):
        if n in p:
            p[n] = a.pop(n)
    args = [a["B"], a["K"], a["V"], a["T"], a["eos"], p["t"], p["max_len"], int(normalize), float(len_penalty)]
    args += [p[n] for n in NAMES[2:]]
    rc = _lib().st5_beam_update(*args, _st())
    torch.cuda.synchronize()
    return rc


LOCKSTEP = {
    # name: (K, B, max_len, min_len, T extra, E per sentence (None: never), dtype, normalize, len_penalty)
    "k1": (1, 3, 130, 1, 9, [20, 66, None], F32, True, 1.0),
    "k4_min70_tight": (4, 5, 131, 70, 2, [10, 64, 100, 115, None], BF16, True, 0.6),
    "k16": (16, 4, 130, 1, 9, [5, 63, 110, None], F32, False, 1.0),
    "k16_min66": (16, 2, 70, 66, 2, [3, None], BF16, True, 1.0),
}


@pytest.mark.parametrize("name", list(LOCKSTEP))
def test_lockstep_search(name):
    K, B, max_len, min_len, extra, E, dtype, normalize, lpen = LOCKSTEP[name]
    V, eos = 81, 2
    T = max_len + extra                   # BeamGraph: max_len + 1 + CHUNK; extra = 2 meets t + 2 <= T with equality
    BK = B * K
    E = [max_len + 10 if e is None else e for e in E]
    logits = Prefix(B, K, V, eos, E, T, dtype, seed=len(name) * 17 + K)
    st = _state(B, K, T, "cuda")
    st["lin"][:, 0] = torch.arange(BK, dtype=torch.int32, device="cuda")
    st["cur_tok"].fill_(eos)
    st["max_len"].fill_(max_len)
    mask = torch.zeros(V)
    mask[1], mask[V - 1], mask[V - 2] = -INF, -INF, -INF
    mnt = _scalars(min_len)[0]
    mask_d = mask.cuda()
    nws = _lib().st5_beam_topk_ws_floats(B, K)
    finished_at = {}
    t = 0
    for t in range(max_len + 1):
        st["t"].fill_(t)
        x = logits(st["lin"].cpu(), st["tok"].cpu(), t)
        cum = st["cur_score"].cpu()
        ws = torch.full((nws,), NAN, device="cuda")
        xd = x.cuda()
        rc = _lib().st5_beam_topk(P(xd), V, DT[dtype], B, K, V, P(st["cur_score"]), P(mask_d), 1.0, eos, P(st["t"]),
                                  P(mnt), P(st["max_len"]), P(st["cand_score"]), P(st["cand_token"]),
                                  P(st["cand_beam"]), P(ws), _st())
        torch.cuda.synchronize()
        assert rc == 0
        n = _beam_n(t, K, V)
        z, bnd = BR.scores(x, cum, mask, 1.0, eos, t, min_len, max_len, K)
        cs, ct, cb = st["cand_score"].cpu(), st["cand_token"].cpu(), st["cand_beam"].cpu()
        before = {k: v.cpu().clone() for k, v in st.items()}
        for s in range(B):
            if before["finished"][s]:
                continue
            same = BR.same_inputs(x, cum, mask, eos, K, s, t)
            w = BR.check_sentence(z[s], bnd[s], cs[s, :n], ct[s, :n], cb[s, :n], V, same, what=f"{name} t={t} s={s}")
            key = f"beam_topk lockstep {'bf16' if dtype == BF16 else 'f32'}"
            REPORT[key] = max(REPORT.get(key, 0.0), w)
        want = {k: v.clone() for k, v in before.items()}
        # (len_penalty is an fp32 argument of the C ABI: 0.6f, not 0.6, is the exponent; with it the arithmetic is the
        # same -- fp32 differences of the same cumulative scores, an fp32 quotient by pow rounded to fp32 -- so every
        # tensor, fin_pos and fin_score included, is compared bit for bit)
        beam_ref.update(want, K, V, eos, normalize, float(np.float32(lpen)))
        assert _update(st, B, K, V, T, eos, normalize, lpen) == 0
        for k in NAMES:
            assert torch.equal(_bits(st[k].cpu()), _bits(want[k])), (name, t, k)
        # a finished sentence's state is left bit-identical
        for s in range(B):
            if before["finished"][s]:
                rs = slice(s * K, (s + 1) * K)
                for k in ("lin", "tok", "score", "ignore", "parent", "cur_tok", "cur_score"):
                    assert torch.equal(_bits(st[k][rs].cpu()), _bits(before[k][rs])), (name, t, s, k)
                for k in ("fin_n", "fin_tok", "fin_pos", "fin_len", "fin_score", "finished"):
                    assert torch.equal(_bits(st[k][s].cpu()), _bits(before[k][s])), (name, t, s, k)
            elif int(st["finished"][s]):
                finished_at[s] = t
        # (ignore fills only when fewer than K of the n candidates are neither eos nor ignored. Each beam offers one
        # eos, so with n = 2K and an empty set at least K are: it stays empty in any search with V > K)
        assert not bool(st["ignore"].any())
        if int(st["stop"][t]):
            break
    STEPS[name] = t
    never = [s for s, e in enumerate(E) if e > max_len]
    assert t == max_len and all(finished_at.get(s) == max_len for s in never), (name, t, finished_at)
    # sentences finish at different steps, and some with hypotheses finalized while others went on
    early = sorted(v for s, v in finished_at.items() if s not in never)
    assert len(set(early)) >= min(2, len(early)) and all(v < max_len for v in early), finished_at
    assert bool((st["fin_n"].cpu() == K).all())
    fl = st["fin_len"].cpu()
    assert int(fl.min()) >= min(min_len, max_len) + 1
    if max_len >= 129:
        assert t >= 129


# ============================================================================================ st5_attn_lineage_fwd
class Lineage:
    """q rows [BQ, W] (q at columns [0, H 64), NaN after); the cache [R, Tbuf, W] with k at block 1 and v at block 2 of
    W = 3 H 64 + 8 columns (block 0 and the tail NaN), finite only in the (row, position) cells some query row's table
    names for an unmasked key; out rows of pitch H 64 + 32 (gaps NaN); probs [BQ, H, Tk] and ws NaN."""

    def __init__(self, q, kc, vc, dtype, Tk, key_pad, rows=None, div=1, cells=None):
        BQ, H = q.shape[0], q.shape[1]
        R, Tbuf = kc.shape[0], kc.shape[1]
        self.BQ, self.H, self.Tk, self.dtype, self.div = BQ, H, Tk, dtype, div
        d = H * 64
        W = 3 * d + 8
        self.W, self.Tbuf = W, Tbuf
        qh = torch.full((BQ, W), NAN)
        qh[:, :d] = q.reshape(BQ, d).float()
        kv = torch.full((R, Tbuf, W), NAN)
        kv[:, :, d:2 * d] = kc.reshape(R, Tbuf, d).float()
        kv[:, :, 2 * d:3 * d] = vc.reshape(R, Tbuf, d).float()
        if cells is not None:
            kv[~cells] = NAN
        self.qb = Flat((BQ, W), dtype)
        self.qb.t.copy_(qh)
        self.kvb = Flat((R, Tbuf, W), dtype)
        self.kvb.t.copy_(kv)
        self.o_bs = d + 32
        self.out = Flat((BQ, self.o_bs), dtype)
        self.probs = Flat((BQ, H, Tk), F32)
        self.ws = Flat((max(1, _lib().st5_attn_decode_ws_floats(BQ, H, Tk, 1)),), F32)
        self.kp = key_pad.cuda().contiguous() if key_pad is not None else None
        self.rows = rows.cuda().contiguous() if rows is not None else None

    def bufs(self):
        return [self.qb, self.kvb, self.out, self.probs, self.ws]

    def run(self, scale=0.125, k_off=0, rows_ld=None, div=None, rows=True):
        from speecht5_b200 import _lib as L
        a = L.AttnLineageArgs()
        b = a.base
        H, d = self.H, self.H * 64
        esz = 4 if self.dtype == F32 else 2
        b.B, b.H, b.Tk, b.dtype = self.BQ, H, self.Tk, DT[self.dtype]
        base = self.kvb.t.data_ptr()
        b.q, b.q_bs = self.qb.t.data_ptr(), self.W
        b.k, b.k_ld, b.k_bs = base + (d + k_off) * esz, self.W, self.Tbuf * self.W
        b.v, b.v_ld, b.v_bs = base + 2 * d * esz, self.W, self.Tbuf * self.W
        b.key_pad = self.kp.data_ptr() if self.kp is not None else None
        b.out, b.o_bs = self.out.t.data_ptr(), self.o_bs
        b.probs, b.scale, b.ws = self.probs.t.data_ptr(), scale, self.ws.t.data_ptr()
        use = self.rows is not None and rows
        a.kv_rows = self.rows.data_ptr() if use else None
        a.kv_rows_ld = (rows_ld if rows_ld is not None else self.rows.shape[1]) if use else 0
        a.kv_div = self.div if div is None else div
        rc = _lib().st5_attn_lineage_fwd(C.byref(a), _st())
        torch.cuda.synchronize()
        return rc

    def out_rows(self):
        o = self.out.t.view(self.BQ, self.o_bs)
        assert bool(torch.isnan(o[:, self.H * 64:].float()).all()), "out: gap between rows written"
        return o[:, :self.H * 64].reshape(self.BQ, self.H, 64)


def _lineage_pad(BQ, Tk, g):
    """Query row 0 all keys, row 1 one key, row 2 none (zeros), row 3 keys 64..127 masked, the rest ragged."""
    L = [Tk, 1, 0] + [int(torch.randint(1, Tk + 1, (1,), generator=g)) for _ in range(BQ - 3)]
    kp = (torch.arange(Tk)[None] >= torch.tensor(L)[:, None]).to(torch.uint8)
    if BQ > 3:
        kp[3] = 0
        kp[3, 64:128] = 1
    return kp


def _check_lineage(name, lg, q, kg, vg, kp):
    f = A.decode_forward(q.double(), kg.double(), vg.double(), scale=0.125, key_pad=kp)
    bnd = A.decode_bounds(f, u=rowops_ref.unit(lg.dtype))
    out = lg.out_rows()
    for b in lg.bufs():
        b.untouched(name)
    A.check(f"lineage {name} out", out.cpu(), f["out"][:, :, 0], bnd["out"], dims="bhc", report=REPORT)
    pr = lg.probs.t.cpu()
    A.check(f"lineage {name} probs", pr, f["P"][:, :, 0], bnd["P"], dims="bhj", report=REPORT)
    return out.clone(), lg.probs.t.clone()


LIN_TK = [1, 63, 64, 65, 129, 600, 1500]


@pytest.mark.parametrize("i,Tk", list(enumerate(LIN_TK)))
@pytest.mark.parametrize("dtype", [F32, BF16])
def test_lineage_self_attention(i, Tk, dtype):
    B, K = 2, 3
    BQ, H = B * K, (1, 12)[i % 2]
    T = Tk + 9                                      # kv_rows_ld > Tk
    g = torch.Generator().manual_seed(50 + i)
    st = _state(B, K, T)
    _random_history(st, K, Tk - 1, g)
    rows = st["lin"].clone()
    R = BQ + 1                                      # row BQ of the cache is all NaN
    rows[:, Tk:] = BQ                               # (valid indices of a NaN row: never read)
    kp = _lineage_pad(BQ, Tk, g)
    q =(torch.randn(BQ, H, 64, generator=g) * math.sqrt(3.0)).to(dtype)
    kc = (torch.randn(R, T, H, 64, generator=g) * math.sqrt(3.0)).to(dtype)
    vc = torch.randn(R, T, H, 64, generator=g).to(dtype)
    j = torch.arange(Tk)
    named = torch.zeros(R, T, dtype=torch.bool)
    live = kp == 0
    named[rows[:, :Tk].long()[live], j[None].expand(BQ, Tk)[live]] = True
    named[BQ] = False
    lg = Lineage(q, kc, vc, dtype, Tk, kp, rows=rows, cells=named)
    assert lg.run() == 0
    kg = kc[rows[:, :Tk].long(), j[None]].permute(0, 2, 1, 3)       # [BQ, H, Tk, 64]
    vg = vc[rows[:, :Tk].long(), j[None]].permute(0, 2, 1, 3)
    kg = torch.where(live[:, None, :, None], kg, torch.zeros_like(kg))
    vg = torch.where(live[:, None, :, None], vg, torch.zeros_like(vg))
    name = f"self {'bf16' if dtype == BF16 else 'f32'}"
    out, pr = _check_lineage(name, lg, q, kg, vg, kp)
    assert bool((out[2] == 0).all()) and bool((pr.view(BQ, H, Tk)[2] == 0).all())
    # a subset of the query rows (B changes): bit-identical rows
    sub = [1, 3] if BQ > 3 else [1]
    lg2 = Lineage(q[sub], kc, vc, dtype, Tk, kp[sub], rows=rows[sub], cells=named)
    assert lg2.run() == 0
    assert torch.equal(_bits(lg2.out_rows()), _bits(out[sub]))
    assert torch.equal(_bits(lg2.probs.t), _bits(pr.view(BQ, H, Tk)[sub]))
    # a wider key span whose extra keys are masked: bit-identical, zero probabilities past Tk
    T2 = Tk + 70
    rows2 = torch.full((BQ, T2 + 3), BQ, dtype=torch.int32)
    rows2[:, :Tk] = rows[:, :Tk]
    kc2 = torch.cat([kc, torch.randn(R, T2 + 3 - T, H, 64, generator=g).to(dtype)], 1)
    vc2 = torch.cat([vc, torch.randn(R, T2 + 3 - T, H, 64, generator=g).to(dtype)], 1)
    named2 = torch.cat([named, torch.zeros(R, T2 + 3 - T, dtype=torch.bool)], 1)
    kp2 = torch.cat([kp, torch.ones(BQ, T2 - Tk, dtype=torch.uint8)], 1)
    lg3 = Lineage(q, kc2, vc2, dtype, T2, kp2, rows=rows2, cells=named2)
    assert lg3.run() == 0
    assert torch.equal(_bits(lg3.out_rows()), _bits(out))
    p3 = lg3.probs.t.view(BQ, H, T2)
    assert torch.equal(_bits(p3[..., :Tk]), _bits(pr.view(BQ, H, Tk)))
    assert bool((p3[..., Tk:] == 0).all())


@pytest.mark.parametrize("i,Tk", list(enumerate(LIN_TK)))
@pytest.mark.parametrize("dtype", [F32, BF16])
def test_lineage_cross_attention_kv_div(i, Tk, dtype):
    """kv_div = K: K query rows per cache row (rows >= B of nothing; positions >= Tk NaN), against the reference and
    bit-identical to kv_div = 1 over a repeat_interleaved cache."""
    B, K = 3, 4
    BQ, H = B * K, (12, 1)[i % 2]
    g = torch.Generator().manual_seed(80 + i)
    kp = _lineage_pad(BQ, Tk, g)
    q = (torch.randn(BQ, H, 64, generator=g) * math.sqrt(3.0)).to(dtype)
    kc = (torch.randn(B, Tk + 5, H, 64, generator=g) * math.sqrt(3.0)).to(dtype)
    vc = torch.randn(B, Tk + 5, H, 64, generator=g).to(dtype)
    cells = torch.zeros(B, Tk + 5, dtype=torch.bool)
    cells[:, :Tk] = (kp == 0).view(B, K, Tk).any(1)
    lg = Lineage(q, kc, vc, dtype, Tk, kp, div=K, cells=cells)
    assert lg.run() == 0
    idx = torch.arange(BQ) // K
    kg, vg = kc[idx, :Tk].permute(0, 2, 1, 3), vc[idx, :Tk].permute(0, 2, 1, 3)
    live = (kp == 0)[:, None, :, None]
    kg, vg = torch.where(live, kg, torch.zeros_like(kg)), torch.where(live, vg, torch.zeros_like(vg))
    out, pr = _check_lineage(f"cross {'bf16' if dtype == BF16 else 'f32'}", lg, q, kg, vg, kp)
    lg2 = Lineage(q, kc.repeat_interleave(K, 0), vc.repeat_interleave(K, 0), dtype, Tk, kp, div=1,
                  cells=cells.repeat_interleave(K, 0))
    assert lg2.run() == 0
    assert torch.equal(_bits(lg2.out_rows()), _bits(out))
    assert torch.equal(_bits(lg2.probs.t), _bits(pr))


@pytest.mark.parametrize("what", ["div0", "rows_div", "rows_ld", "k_misaligned"])
@pytest.mark.parametrize("dtype", [F32, BF16])
def test_lineage_rejections_leave_buffers_untouched(what, dtype):
    B, K, Tk, H = 2, 2, 100, 2
    BQ, T = B * K, Tk + 4
    g = torch.Generator().manual_seed(9)
    st = _state(B, K, T)
    _random_history(st, K, Tk - 1, g)
    q = torch.randn(BQ, H, 64, generator=g).to(dtype)
    kc = torch.randn(BQ, T, H, 64, generator=g).to(dtype)
    vc = torch.randn(BQ, T, H, 64, generator=g).to(dtype)
    lg = Lineage(q, kc, vc, dtype, Tk, _lineage_pad(BQ, Tk, g), rows=st["lin"])
    snaps = [b.flat.clone() for b in lg.bufs()]
    kw = {"div0": dict(div=0, rows=False), "rows_div": dict(div=K), "rows_ld": dict(rows_ld=Tk - 1),
          "k_misaligned": dict(k_off=1)}[what]
    want = -6 if what == "k_misaligned" else -2
    assert lg.run(**kw) == want
    assert all(torch.equal(_bits(b.flat), _bits(s)) for b, s in zip(lg.bufs(), snaps)), what


UPDATE_REJECT = [("T1", -2), ("K0", -2), ("K17", -2), ("B0", -2), ("V=K", -2)] + [(f"null:{n}", -3) for n in NAMES]


@pytest.mark.parametrize("what,want", UPDATE_REJECT)
def test_update_rejections_leave_buffers_untouched(what, want):
    B, K, T, V = 3, 4, 32, 60
    g = torch.Generator().manual_seed(6)
    st = _state(B, K, T)
    _random_history(st, K, 5, g)
    st["t"][0], st["max_len"][0] = 5, 20
    st["cand_score"] = torch.sort(-torch.rand(B, 2 * K, generator=g) * 5, descending=True).values
    st["cand_token"] = torch.randint(4, V, (B, 2 * K), generator=g, dtype=torch.int32)
    st["cand_beam"] = torch.randint(0, K, (B, 2 * K), generator=g, dtype=torch.int32)
    st = {k: v.cuda() for k, v in st.items()}
    snaps = {k: v.clone() for k, v in st.items()}
    over = {"T1": dict(T=1), "K0": dict(K=0), "K17": dict(K=17), "B0": dict(B=0), "V=K": dict(V=K)}.get(what, {})
    if what.startswith("null:"):
        over = {what[5:]: None}
    assert _update(st, B, K, V, T, 2, True, 1.0, over) == want
    for k in st:
        assert torch.equal(_bits(st[k]), _bits(snaps[k])), (what, k)
