"""-m gpu: every attention entry point of include/speecht5_b200.h called directly (kernels.attn_*), against the fp64
statement of tests/attention_ref.py with ELEMENTWISE bounds, on buffers laid out here with NaN sentinels everywhere the
contract does not let a kernel read or write:
  - q / k / v sit in one column block of wider buffers (the other blocks NaN) with NaN gap rows between utterances;
    out / dq / dk / dv likewise (o_ld > H*64), every buffer with NaN guard zones before and after;
  - psave, probs, ds, delta and dq_acc start NaN: scratch must be written before it is read, psave must hold zeros in
    every column the backward reads (dead causal chunks and [Tk, p_ld) included), heads >= probs_heads stay untouched;
  - the padding columns [Tk, p_ld) of dprobs_ext and its heads >= ext_heads are NaN (the backward does not read them);
  - dpe_k starts non-zero (the row backward adds to it).
Inputs have peaked scores (std ~3) so that one wrong key moves the output past the bound; the relative-position probe
sets k = 0 so that every score is a table entry. Dropout masks (psave sign bits) are compared with tests/dropout_ref.py.
The largest err / bound of every entry point is printed at the end of the module (run with -s)."""
import math

import pytest
import torch

import attention_ref as R
import dropout_ref as D

pytestmark = pytest.mark.gpu

NAN = float("nan")
G = 64  # guard elements before and after every buffer (16-byte aligned offsets for every dtype)
SEED, OFFSET = 1234, 7
SCALE = 0.125
REPORT = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if REPORT:
        print("\nlargest err / bound per entry point:")
        for k in sorted(REPORT):
            print(f"  {k:40s} {REPORT[k]:.3g}")


def _r8(x):
    return (x + 7) // 8 * 8


class Rows:
    """Logical [B][T][H*64] at element b*bs + t*ld + col0 + h*64 + c of a NaN buffer (gap rows, other column blocks
    and guard zones stay NaN)."""

    def __init__(self, B, T, H, dtype, ld, col0=0, gap=3):
        self.B, self.T, self.H, self.d, self.ld, self.col0, self.gap = B, T, H, H * 64, ld, col0, gap
        self.bs = (T + gap) * ld
        self.flat = torch.full((2 * G + B * self.bs,), NAN, dtype=dtype, device="cuda")
        self.inside = torch.zeros(self.flat.numel(), dtype=torch.bool, device="cuda")
        self._region(self.inside).fill_(True)

    def _region(self, t):
        return t[G:G + self.B * self.bs].view(self.B, self.T + self.gap, self.ld)[:, :self.T,
                                                                               self.col0:self.col0 + self.d]

    @property
    def ptr(self):
        return self.flat[G + self.col0:]

    def set(self, x):  # x [B, H, T, 64]
        self._region(self.flat).copy_(x.permute(0, 2, 1, 3).reshape(self.B, self.T, self.d))

    def get(self):
        return self._region(self.flat).reshape(self.B, self.T, self.H, 64).permute(0, 2, 1, 3).cpu()

    def untouched(self, what):
        bad = ~torch.isnan(self.flat[~self.inside].float())
        assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements written outside the logical region"


class Flat:
    """A contiguous [shape] tensor inside a NaN buffer with guard zones."""

    def __init__(self, shape, dtype, fill=NAN):
        n = math.prod(shape)
        self.shape = shape
        self.flat = torch.full((2 * G + n,), NAN, dtype=dtype, device="cuda")
        self.t = self.flat[G:G + n].view(shape)
        if fill is not None and not math.isnan(fill):
            self.t.fill_(fill)

    @property
    def ptr(self):
        return self.t

    def get(self):
        return self.t.cpu()

    def untouched(self, what):
        g = torch.cat([self.flat[:G], self.flat[-G:]]).float()
        assert bool(torch.isnan(g).all()), f"{what}: guard zone written"


def _kernels():
    from speecht5_b200 import _lib
    from speecht5_b200 import kernels as K
    return K, _lib


def _key_pad(pad, B, Tk):
    """None, or ragged lengths: utterance 0 full, utterance 1 one key, the rest about half."""
    if not pad:
        return None
    kp = torch.zeros(B, Tk, dtype=torch.bool)
    for b in range(1, B):
        kp[b, (1 if b == 1 else Tk // 2 + 1):] = True
    return kp


def _masked_keys(f):
    """[B, Tk] bool: keys no query row of utterance b sees (their dK / dV must be exactly zero)."""
    return ~f["ok"].any(2)[:, 0]


def _layout(B, H, Tq, Tk, dtype):
    d = H * 64
    qb = Rows(B, Tq, H, dtype, ld=3 * d, col0=d)       # q at block 1 of 3
    kb = Rows(B, Tk, H, dtype, ld=3 * d, col0=0)       # k at block 0, v at block 2 (the middle block stays NaN)
    vb = Rows(B, Tk, H, dtype, ld=3 * d, col0=2 * d)
    return qb, kb, vb


def _base_args(K, B, H, Tq, Tk, dtype_id, qb, kb, vb, out, causal, maxpos, pe, kp, drop, p_ld):
    return dict(B=B, H=H, Tq=Tq, Tk=Tk, dtype=dtype_id, causal=int(causal), maxpos=maxpos if pe is not None else 0,
                q=qb.ptr, q_ld=qb.ld, q_bs=qb.bs, k=kb.ptr, k_ld=kb.ld, k_bs=kb.bs, v=vb.ptr, v_ld=vb.ld, v_bs=vb.bs,
                key_pad=kp, pe_k=pe, out=out.ptr, o_ld=out.ld, o_bs=out.bs, p_ld=p_ld, scale=SCALE, drop_p=drop,
                seed=SEED, offset=OFFSET)


def _check_probs(name, got, f, bnd, p_ld, Tk, heads=None):
    """fp32 (or bf16) probabilities [B, H, Tq, p_ld]: within bound on [.., :Tk], zero on masked keys and [Tk, p_ld);
    heads >= `heads` untouched (NaN)."""
    H = got.shape[1]
    nh = heads if heads else H
    g = got[:, :nh].double()
    R.check(name, g[..., :Tk], f["P"][:, :nh], bnd[:, :nh], report=REPORT)
    if p_ld > Tk:
        assert bool((g[..., Tk:] == 0).all()), f"{name}: columns [Tk, p_ld) not zero"
    if nh < H:
        assert bool(torch.isnan(got[:, nh:].float()).all()), f"{name}: heads >= probs_heads written"


# ============================================================================= wgmma forward (resident / streaming)
def run_fused(entry, B, H, Tq, Tk, *, causal=False, maxpos=0, probe=False, pad=False, drop=0.0, want_probs=False,
              p_ld=None, probs_heads=0, ext_heads=None, with_psave=True, bwd=True, seed=0):
    K, _lib = _kernels()
    q, k, v, pe = R.make_inputs(B, H, Tq, Tk, seed=seed, maxpos=maxpos, probe=probe)
    pe_bf = pe.to(torch.bfloat16) if pe is not None else None
    kp = _key_pad(pad, B, Tk)
    p_ld = p_ld or _r8(Tk)
    qb, kb, vb = _layout(B, H, Tq, Tk, torch.bfloat16)
    for buf, x in ((qb, q), (kb, k), (vb, v)):
        buf.set(x.cuda())
    d = H * 64
    out = Rows(B, Tq, H, torch.bfloat16, ld=d + 16, gap=2)
    psave = Flat((B, H, Tq, p_ld), torch.bfloat16) if with_psave else None
    inv_l = Flat((B, H, Tq), torch.float32) if with_psave else None
    o32 = Flat((B, Tq, d), torch.float32) if with_psave else None
    lse = Flat((B, H, Tq), torch.float32)
    probs = Flat((B, H, Tq, p_ld), torch.float32) if (want_probs or ext_heads is not None) else None
    kp_dev = kp.to(torch.uint8).cuda() if kp is not None else None
    pe_dev = pe_bf.cuda() if pe_bf is not None else None
    kw = _base_args(K, B, H, Tq, Tk, _lib.BF16, qb, kb, vb, out, causal, maxpos, pe_dev, kp_dev, drop, p_ld)
    a = K.attn_args(**kw, probs=probs.ptr if probs is not None else None, probs_dtype=_lib.F32,
                    probs_heads=probs_heads)
    fwd = K.attn_flash_fwd if entry == "flash" else K.attn_fused_fwd
    fwd(a, lse.ptr, psave.ptr if psave else None, inv_l.ptr if inv_l else None, o32.ptr if o32 else None)
    torch.cuda.synchronize()

    f = R.forward(q, k, v, scale=SCALE, pe=pe_bf, maxpos=maxpos, causal=causal, key_pad=kp, drop_p=drop, seed=SEED,
                  offset=OFFSET)
    bnd = R.bounds(f, u=R.U_BF16, C=R.C_BF16)
    n = f"{entry}_fwd"
    R.check(f"{n} out", out.get(), f["out"], bnd["out"], "bhic", REPORT)
    out.untouched(f"{n} out")
    R.check(f"{n} lse", lse.get(), f["lse"], bnd["lse"], "bhi", REPORT)
    lse.untouched(f"{n} lse")
    if probs is not None:
        bP = R.bounds(f, u=R.U_F32, C=R.C_F32)["P"]
        _check_probs(f"{n} probs", probs.get(), f, bP, p_ld, Tk, probs_heads)
        probs.untouched(f"{n} probs")
    if with_psave:
        R.check(f"{n} inv_l", inv_l.get(), f["inv_l"], bnd["inv_l"], "bhi", REPORT)
        R.check(f"{n} out_f32", o32.get().view(B, Tq, H, 64).permute(0, 2, 1, 3), f["out"], bnd["out"], "bhic",
                REPORT)
        for t, w in ((inv_l, "inv_l"), (o32, "out_f32"), (psave, "psave")):
            t.untouched(f"{n} {w}")
        ps = psave.get()
        # the columns the backward reads: every key block of the row's tile up to p_ld (causal: blocks <= the tile's)
        reach = torch.full((Tq,), p_ld)
        if causal:
            reach = torch.minimum(reach, (torch.arange(Tq) // 64 + 1) * 64)
        cols = torch.arange(p_ld)[None, :] < reach[:, None]          # [Tq, p_ld]
        okp = torch.zeros(B, H, Tq, p_ld, dtype=torch.bool)
        okp[..., :Tk] = f["ok"]
        region = ps[:, :, :, :][..., :p_ld]
        live = region[cols.expand(B, H, Tq, p_ld) & okp].double()
        R.check(f"{n} psave", live.abs(), f["e"][okp[..., :Tk]], bnd["e"][okp[..., :Tk]], "n", REPORT)
        dead = region[cols.expand(B, H, Tq, p_ld) & ~okp].float()
        assert bool((dead == 0).all()), f"{n} psave: {int((dead != 0).sum())} non-zero (or NaN) masked / padding " \
                                        f"entries the backward reads"
        if drop > 0:  # dropout decision in the sign bit of every element that takes part
            sign = torch.signbit(region[..., :Tk].float())
            want = ~f["keep"]
            bad = (sign != want) & f["ok"]
            assert not bool(bad.any()), f"{n} psave: sign bit != dropout_ref at {tuple(torch.nonzero(bad)[0].tolist())}"
    if not bwd:
        return
    run_fused_bwd(K, _lib, f, q, k, v, pe_bf, kp_dev, qb, kb, vb, out, psave, inv_l, o32, probs, kw, p_ld,
                  ext_heads, seed)


def run_fused_bwd(K, _lib, f, q, k, v, pe_bf, kp_dev, qb, kb, vb, out, psave, inv_l, o32, probs, kw, p_ld,
                  ext_heads, seed):
    B, H, Tq, Tk = kw["B"], kw["H"], kw["Tq"], kw["Tk"]
    d = H * 64
    gen = torch.Generator().manual_seed(seed + 100)
    dO = torch.randn(B, H, Tq, 64, generator=gen).to(torch.bfloat16)
    dout = Rows(B, Tq, H, torch.bfloat16, ld=out.ld, gap=2)
    dout.set(dO.cuda())
    ext = None
    dpx = None
    if ext_heads is not None:
        eh = ext_heads if 0 < ext_heads < H else H
        ext = torch.zeros(B, H, Tq, Tk)
        ext[:, :eh] = torch.randn(B, eh, Tq, Tk, generator=gen) * 4.0
        dpx = Flat((B, H, Tq, p_ld), torch.float32)
        dpx.t[:, :eh, :, :Tk] = ext[:, :eh].cuda()  # heads >= ext_heads and columns [Tk, p_ld) stay NaN
    dq, dk, dv = (Rows(b.B, b.T, b.H, torch.bfloat16, ld=b.ld, col0=b.col0) for b in (qb, kb, vb))
    delta = Flat((B, H, Tq), torch.float32)
    dq_acc = Flat((B, Tq, d), torch.float32)
    ds = Flat((B, H, Tq, p_ld), torch.bfloat16) if pe_bf is not None else None
    a = K.attn_args(**kw, probs=probs.ptr if (probs is not None and dpx is not None) else None,
                    probs_dtype=_lib.F32, dout=dout.ptr, dprobs_ext=dpx.ptr if dpx is not None else None,
                    ds=ds.ptr if ds is not None else None, dq=dq.ptr, dk=dk.ptr, dv=dv.ptr)
    K.attn_fused_bwd(a, psave.ptr, inv_l.ptr, o32.ptr, delta.ptr, dq_acc.ptr,
                     ext_heads=ext_heads if ext_heads is not None else 0)
    torch.cuda.synchronize()
    g = R.backward(f, dO, ext)
    bnd = R.bounds(f, g, u=R.U_BF16, C=R.C_BF16)
    n = "fused_bwd"
    dq_name = "dQ_k" if pe_bf is not None else "dQ"
    R.check(f"{n} dq", dq.get(), g[dq_name], bnd[dq_name], "bhic", REPORT)
    R.check(f"{n} dk", dk.get(), g["dK"], bnd["dK"], "bhjc", REPORT)
    R.check(f"{n} dv", dv.get(), g["dV"], bnd["dV"], "bhjc", REPORT)
    for t, w in ((dq, "dq"), (dk, "dk"), (dv, "dv")):
        t.untouched(f"{n} {w}")
    mk = _masked_keys(f)
    if bool(mk.any()):
        for t, w in ((dk, "dk"), (dv, "dv")):
            got = t.get().permute(0, 2, 1, 3)[mk]
            assert bool((got == 0).all()), f"{n} {w}: masked keys with a non-zero gradient"
    if ds is not None:
        dsg = ds.get()
        R.check(f"{n} ds", dsg[..., :Tk], g["dS"], bnd["dS"], "bhij", REPORT)
        assert bool((dsg[..., Tk:].float() == 0).all()), f"{n} ds: columns [Tk, p_ld) not zero"
        ds.untouched(f"{n} ds")
    delta.untouched(f"{n} delta")
    dq_acc.untouched(f"{n} dq_acc")


FUSED_CASES = [
    # resident kernel: Tk <= 320
    dict(entry="fused", B=2, H=2, Tq=1, Tk=1),
    dict(entry="fused", B=2, H=2, Tq=63, Tk=63, drop=0.2),
    dict(entry="fused", B=2, H=2, Tq=64, Tk=64),
    dict(entry="fused", B=2, H=2, Tq=65, Tk=65, pad=True),
    dict(entry="fused", B=3, H=2, Tq=129, Tk=129, pad=True, drop=0.2),
    dict(entry="fused", B=2, H=2, Tq=320, Tk=320),
    dict(entry="fused", B=2, H=2, Tq=129, Tk=129, causal=True, drop=0.2),
    dict(entry="fused", B=2, H=2, Tq=70, Tk=320, pad=True),
    dict(entry="fused", B=2, H=2, Tq=64, Tk=64, maxpos=64, probe=True),
    dict(entry="fused", B=3, H=2, Tq=100, Tk=100, maxpos=100, probe=True, pad=True, drop=0.2),
    dict(entry="fused", B=1, H=2, Tq=160, Tk=160, maxpos=160, probe=True),
    dict(entry="fused", B=2, H=3, Tq=129, Tk=129, want_probs=True, ext_heads=0),
    dict(entry="fused", B=2, H=3, Tq=129, Tk=129, want_probs=True, probs_heads=2, ext_heads=2, drop=0.2),
    # streaming kernel: any length
    dict(entry="flash", B=2, H=2, Tq=65, Tk=65),
    dict(entry="flash", B=2, H=2, Tq=321, Tk=321, drop=0.2),
    dict(entry="flash", B=2, H=2, Tq=130, Tk=499, pad=True),
    dict(entry="flash", B=1, H=2, Tq=512, Tk=512),
    dict(entry="flash", B=1, H=2, Tq=513, Tk=513, pad=True),
    dict(entry="flash", B=1, H=2, Tq=781, Tk=781, drop=0.2),
    dict(entry="flash", B=2, H=2, Tq=130, Tk=130, causal=True, drop=0.2),
    dict(entry="flash", B=1, H=2, Tq=500, Tk=500, causal=True),
    dict(entry="flash", B=2, H=2, Tq=70, Tk=200, causal=True),
    dict(entry="flash", B=2, H=2, Tq=65, Tk=65, maxpos=8, probe=True),
    dict(entry="flash", B=2, H=2, Tq=199, Tk=199, maxpos=48, probe=True, drop=0.2),
    dict(entry="flash", B=2, H=2, Tq=199, Tk=199, maxpos=64, probe=True),
    dict(entry="flash", B=1, H=2, Tq=781, Tk=781, maxpos=160, pad=False),
    dict(entry="flash", B=2, H=2, Tq=199, Tk=199, maxpos=64, pad=True),
    dict(entry="flash", B=2, H=3, Tq=313, Tk=313, want_probs=True, p_ld=313, with_psave=False, bwd=False),
    dict(entry="flash", B=2, H=3, Tq=100, Tk=313, want_probs=True, p_ld=316, with_psave=False, bwd=False,
         probs_heads=2),
    dict(entry="flash", B=2, H=3, Tq=130, Tk=130, causal=True, want_probs=True, probs_heads=2, ext_heads=2),
    dict(entry="flash", B=2, H=3, Tq=200, Tk=499, want_probs=True, ext_heads=0, drop=0.2),
]


def _id(c):
    return "-".join(f"{k}{v}" for k, v in c.items() if k != "entry" and v not in (False, None)) + f"-{c['entry']}"


@pytest.mark.parametrize("case", FUSED_CASES, ids=[_id(c) for c in FUSED_CASES])
def test_wgmma_forward_and_fused_backward(cuda, case):
    c = dict(case)
    run_fused(c.pop("entry"), c.pop("B"), c.pop("H"), c.pop("Tq"), c.pop("Tk"), **c)


def test_flash_forward_longest_utterance(cuda):
    """7,999 encoder frames with clipped relative positions (speaker identification on a 160 s utterance): forward only,
    the first, one middle and the last query tile against the fp64 statement of those rows."""
    K, _lib = _kernels()
    B, H, T, maxpos = 1, 1, 7999, 160
    q, k, v, pe = R.make_inputs(B, H, T, T, seed=5, maxpos=maxpos)
    pe_bf = pe.to(torch.bfloat16)
    qb, kb, vb = _layout(B, H, T, T, torch.bfloat16)
    for buf, x in ((qb, q), (kb, k), (vb, v)):
        buf.set(x.cuda())
    out = Rows(B, T, H, torch.bfloat16, ld=64 + 16, gap=2)
    kw = _base_args(K, B, H, T, T, _lib.BF16, qb, kb, vb, out, False, maxpos, pe_bf.cuda(), None, 0.0, _r8(T))
    K.attn_flash_fwd(K.attn_args(**kw), None)
    torch.cuda.synchronize()
    got = out.get()
    out.untouched("flash_fwd T=7999 out")
    for r0 in (0, 62 * 64, 124 * 64):
        rows = torch.arange(r0, min(r0 + 64, T))
        f = R.forward(q[:, :, rows], k, v, scale=SCALE, pe=pe_bf, maxpos=maxpos, rows=rows)
        bnd = R.bounds(f, u=R.U_BF16, C=R.C_BF16)
        R.check("flash_fwd out (T=7999)", got[:, :, rows], f["out"], bnd["out"], "bhic", REPORT)


# ============================================================================= row kernels (fp32 parity / bf16)
ROW_CASES = [
    dict(B=2, H=2, Tq=1, Tk=1),
    dict(B=3, H=2, Tq=65, Tk=65, pad=True, drop=0.2),
    dict(B=2, H=2, Tq=130, Tk=130, causal=True, drop=0.2, ext=True),
    dict(B=2, H=2, Tq=70, Tk=200, causal=True),
    dict(B=2, H=2, Tq=100, Tk=313, pad=True, ext=True),
    dict(B=2, H=2, Tq=199, Tk=199, maxpos=64, probe=True),
    dict(B=1, H=2, Tq=781, Tk=781, maxpos=160, drop=0.2),
    dict(B=2, H=2, Tq=37, Tk=37, maxpos=8, probe=True, pad=True),
]


@pytest.mark.parametrize("types", ["f32-f32", "bf16-bf16", "bf16-f32"])
@pytest.mark.parametrize("case", ROW_CASES, ids=[_id(dict(c, entry="row")) for c in ROW_CASES])
def test_row_kernels_forward_and_backward(cuda, case, types):
    K, _lib = _kernels()
    c = dict(case)
    B, H, Tq, Tk = c["B"], c["H"], c["Tq"], c["Tk"]
    maxpos, causal, drop = c.get("maxpos", 0), c.get("causal", False), c.get("drop", 0.0)
    dt, pdt = (torch.float32 if t == "f32" else torch.bfloat16 for t in types.split("-"))
    q, k, v, pe = R.make_inputs(B, H, Tq, Tk, seed=2, maxpos=maxpos, probe=c.get("probe", False), dtype=dt)
    kp = _key_pad(c.get("pad"), B, Tk)
    p_ld = _r8(Tk) + 8
    qb, kb, vb = _layout(B, H, Tq, Tk, dt)
    for buf, x in ((qb, q), (kb, k), (vb, v)):
        buf.set(x.cuda())
    d = H * 64
    out = Rows(B, Tq, H, dt, ld=d + 16, gap=2)
    probs = Flat((B, H, Tq, p_ld), pdt)
    kp_dev = kp.to(torch.uint8).cuda() if kp is not None else None
    pe_dev = pe.cuda() if pe is not None else None
    did = _lib.F32 if dt == torch.float32 else _lib.BF16
    kw = _base_args(K, B, H, Tq, Tk, did, qb, kb, vb, out, causal, maxpos, pe_dev, kp_dev, drop, p_ld)
    kw["probs_dtype"] = _lib.F32 if pdt == torch.float32 else _lib.BF16
    K.attn_fwd(K.attn_args(**kw, probs=probs.ptr))
    torch.cuda.synchronize()
    f = R.forward(q, k, v, scale=SCALE, pe=pe, maxpos=maxpos, causal=causal, key_pad=kp, drop_p=drop, seed=SEED,
                  offset=OFFSET)
    u = R.U_F32 if types == "f32-f32" else R.U_BF16
    C = R.C_F32 if types == "f32-f32" else R.C_BF16
    n = f"attn_fwd[{types}]"
    bnd = R.bounds(f, u=u, C=C)
    R.check(f"{n} out", out.get(), f["out"], bnd["out"], "bhic", REPORT)
    out.untouched(f"{n} out")
    bP = R.bounds(f, u=R.U_F32 if pdt == torch.float32 else R.U_BF16, C=C)["P"]
    _check_probs(f"{n} probs", probs.get(), f, bP, p_ld, Tk)
    probs.untouched(f"{n} probs")

    gen = torch.Generator().manual_seed(7)
    dO = torch.randn(B, H, Tq, 64, generator=gen).to(dt)
    dout = Rows(B, Tq, H, dt, ld=out.ld, gap=2)
    dout.set(dO.cuda())
    ext, dpx = None, None
    if c.get("ext"):
        ext = torch.randn(B, H, Tq, Tk, generator=gen) * 4.0
        dpx = Flat((B, H, Tq, p_ld), torch.float32)
        dpx.t[..., :Tk] = ext.cuda()
    dq, dk, dv = (Rows(b.B, b.T, b.H, dt, ld=b.ld, col0=b.col0) for b in (qb, kb, vb))
    ds = Flat((B, H, Tq, p_ld), torch.float32)
    dpe0 = torch.randn(2 * maxpos, 64, generator=gen) if maxpos else None
    dpe = Flat((2 * maxpos, 64), torch.float32) if maxpos else None
    if maxpos:
        dpe.t.copy_(dpe0.cuda())
    K.attn_bwd(K.attn_args(**kw, probs=probs.ptr, dout=dout.ptr, dprobs_ext=dpx.ptr if dpx else None, ds=ds.ptr,
                           dq=dq.ptr, dk=dk.ptr, dv=dv.ptr, dpe_k=dpe.ptr if dpe else None))
    torch.cuda.synchronize()
    g = R.backward(f, dO, ext)
    bnd = R.bounds(f, g, u=u, C=C)
    n = f"attn_bwd[{types}]"
    R.check(f"{n} dq", dq.get(), g["dQ"], bnd["dQ"], "bhic", REPORT)
    R.check(f"{n} dk", dk.get(), g["dK"], bnd["dK"], "bhjc", REPORT)
    R.check(f"{n} dv", dv.get(), g["dV"], bnd["dV"], "bhjc", REPORT)
    for t, w in ((dq, "dq"), (dk, "dk"), (dv, "dv"), (ds, "ds")):
        t.untouched(f"{n} {w}")
    mk = _masked_keys(f)
    for t, w in ((dk, "dk"), (dv, "dv")):
        assert bool((t.get().permute(0, 2, 1, 3)[mk] == 0).all()), f"{n} {w}: masked keys with a non-zero gradient"
    if maxpos:  # dpe_k += the table gradient
        R.check(f"{n} dpe (+=)", dpe.get().double() - dpe0.double(), g["dPE"], bnd["dPE"] + 2.0 ** -23 * dpe0.abs(),
                "rc", REPORT)
        dpe.untouched(f"{n} dpe")


# ============================================================================= tensor-core route row kernels
TC_CASES = [(1, 3, 8), (64, 64, 8), (313, 313, 160), (512, 512, 160), (313, 100, 8)]  # (Tk, Tq, maxpos)


def _tc_inputs(B, H, Tq, Tk, maxpos, seed):
    q, k, v, pe = R.make_inputs(B, H, Tq, Tk, seed=seed, maxpos=maxpos)
    S = (SCALE * (q.double() @ k.double().transpose(-1, -2))).float()
    QP = (SCALE * (q.double() @ pe.to(torch.bfloat16).double().T)).float()
    return S, QP


@pytest.mark.parametrize("alias", [False, True])
@pytest.mark.parametrize("drop", [0.0, 0.2])
@pytest.mark.parametrize("rpe", [False, True])
@pytest.mark.parametrize("Tk,Tq,maxpos", TC_CASES)
def test_tc_softmax_and_ds(cuda, Tk, Tq, maxpos, rpe, drop, alias):
    K, _lib = _kernels()
    B, H = 2, 2
    causal = not rpe and Tq == Tk
    p_ld = _r8(Tk)
    S, QP = _tc_inputs(B, H, Tq, Tk, maxpos, seed=Tk)
    kp = _key_pad(True, B, Tk) if Tk > 1 else None
    s_buf = Flat((B, H, Tq, p_ld), torch.float32)
    s_buf.t[..., :Tk] = S.cuda()  # padding columns stay NaN: the kernel reads keys < Tk only
    qp_buf = Flat((B, H, Tq, 2 * maxpos), torch.float32)
    qp_buf.t.copy_(QP.cuda())
    P = Flat((B, H, Tq, p_ld), torch.bfloat16)
    probs = s_buf if alias else Flat((B, H, Tq, p_ld), torch.float32)
    Pd = Flat((B, H, Tq, p_ld), torch.bfloat16)
    kp_dev = kp.to(torch.uint8).cuda() if kp is not None else None
    K.attn_softmax_fwd(s_buf.ptr, qp_buf.ptr if rpe else None, kp_dev, P.ptr, probs.ptr, Pd.ptr, B, H, Tq, Tk, p_ld,
                       causal, maxpos, drop, SEED, OFFSET)
    torch.cuda.synchronize()
    s64 = S.double()
    if rpe:
        s64 = s64 + torch.gather(QP.double(), 3, R.rel_index(Tq, Tk, maxpos).expand(B, H, Tq, Tk))
    ok = R.valid_mask(B, Tq, Tk, causal, kp).expand(B, H, Tq, Tk)
    s64 = s64.masked_fill(~ok, -math.inf)
    Pref = torch.softmax(s64, -1)
    sa = torch.where(ok, s64.abs(), torch.zeros_like(s64))
    EP = Pref * 64 * 2.0 ** -24 * (sa + sa.amax(-1, keepdim=True) + 4)
    f = dict(P=Pref)
    n = "softmax_fwd"
    _check_probs(f"{n} probs_f32", probs.get(), f, EP + 2.0 ** -60, p_ld, Tk)
    _check_probs(f"{n} P", P.get(), f, EP + R.U_BF16 * Pref + 2.0 ** -60, p_ld, Tk)
    keep = R.keep_mask(B, H, Tq, Tk, drop, SEED, OFFSET)
    pk = P.get().double()[..., :Tk]
    pd_ref = pk * keep * D.drop_scale(drop)
    R.check(f"{n} dropout(P)", Pd.get()[..., :Tk], pd_ref, R.U_BF16 * pd_ref + 2.0 ** -60, "bhij", REPORT)
    assert bool((Pd.get()[..., Tk:].float() == 0).all()), f"{n} dropout(P): columns [Tk, p_ld) not zero"
    for t, w in ((P, "P"), (Pd, "Pd"), (probs, "probs")):
        t.untouched(f"{n} {w}")

    # ---- dS from the P just written
    gen = torch.Generator().manual_seed(Tk + 1)
    dP = torch.randn(B, H, Tq, Tk, generator=gen) * 8.0
    dP_buf = Flat((B, H, Tq, p_ld), torch.float32)
    dP_buf.t[..., :Tk] = dP.cuda()
    for with_ext in (False, True):
        ext = torch.randn(B, H, Tq, Tk, generator=gen) * 4.0
        ext_buf = Flat((B, H, Tq, p_ld), torch.float32)
        ext_buf.t[..., :Tk] = ext.cuda()
        dS = Flat((B, H, Tq, p_ld), torch.bfloat16)
        Pd2 = Flat((B, H, Tq, p_ld), torch.bfloat16)
        K.attn_ds(P.ptr, dP_buf.ptr, ext_buf.ptr if with_ext else None, dS.ptr, Pd2.ptr, B, H, Tq, Tk, p_ld, drop,
                  SEED, OFFSET)
        torch.cuda.synchronize()
        dPk = dP.double() * keep * D.drop_scale(drop) + (ext.double() if with_ext else 0.0)
        delta = (pk * dPk).sum(-1, keepdim=True)
        ref = pk * (dPk - delta)
        bS = (R.C_F32 * 2.0 ** -20 * pk * (dPk.abs() + (pk * dPk.abs()).sum(-1, keepdim=True))
              + R.U_BF16 * ref.abs() + 2.0 ** -60)
        m = f"ds[ext={int(with_ext)}]"
        R.check(f"{m} dS", dS.get()[..., :Tk], ref, bS, "bhij", REPORT)
        R.check(f"{m} dropout(P)", Pd2.get()[..., :Tk], pd_ref, R.U_BF16 * pd_ref + 2.0 ** -60, "bhij", REPORT)
        for t, w in ((dS, "dS"), (Pd2, "Pd")):
            assert bool((t.get()[..., Tk:].float() == 0).all()), f"{m} {w}: columns [Tk, p_ld) not zero"
            t.untouched(f"{m} {w}")


@pytest.mark.parametrize("misalign", [False, True])
@pytest.mark.parametrize("h_major", [False, True])
@pytest.mark.parametrize("Tk,Tq,maxpos", TC_CASES)
def test_tc_dqp_scatter(cuda, Tk, Tq, maxpos, h_major, misalign):
    K, _lib = _kernels()
    B, H = 2, 3
    p_ld = _r8(Tk)
    gen = torch.Generator().manual_seed(Tk * 7 + maxpos)
    dS = torch.randn(B, H, Tq, Tk, generator=gen).to(torch.bfloat16)
    ds_buf = Flat((B, H, Tq, p_ld), torch.bfloat16)
    ds_buf.t[..., :Tk] = dS.cuda()
    R2 = 2 * maxpos
    n_out = B * H * Tq * R2
    # misalign: the output starts 2 bytes off a 16-byte boundary (the kernel's scalar store path)
    out_flat = torch.full((2 * G + n_out + 1,), NAN, dtype=torch.bfloat16, device="cuda")
    o0 = G + (1 if misalign else 0)
    out = out_flat[o0:o0 + n_out]
    K.attn_dqp_scatter(ds_buf.ptr, out, B, H, Tq, Tk, p_ld, maxpos, h_major=h_major)
    torch.cuda.synchronize()
    ref = R.scatter_qp(dS.double(), maxpos)
    bnd = R.U_BF16 * ref.abs() + 2.0 ** -20 * R.scatter_qp(dS.double().abs(), maxpos) + 2.0 ** -60
    if h_major:
        ref, bnd = R.head_major(ref), R.head_major(bnd)
    got = out.cpu().view(*ref.shape)
    R.check(f"dqp_scatter[h_major={int(h_major)}]", got, ref, bnd, "xyir", REPORT)
    rest = torch.cat([out_flat[:o0], out_flat[o0 + n_out:]]).float()
    assert bool(torch.isnan(rest).all()), "dqp_scatter: written outside [rows, 2 maxpos]"


# ============================================================================= rejected configurations
def test_rejected_configurations_leave_buffers_untouched(cuda):
    """Argument checks return an error before any launch: the NaN output buffers stay NaN."""
    K, _lib = _kernels()

    def fused_args(B, H, Tq, Tk, maxpos=0, p_ld=None, probs_dtype=None):
        q, k, v, pe = R.make_inputs(B, H, Tq, Tk, maxpos=maxpos)
        qb, kb, vb = _layout(B, H, Tq, Tk, torch.bfloat16)
        for buf, x in ((qb, q), (kb, k), (vb, v)):
            buf.set(x.cuda())
        out = Rows(B, Tq, H, torch.bfloat16, ld=H * 64 + 16, gap=2)
        pe_dev = pe.to(torch.bfloat16).cuda() if pe is not None else None
        p_ld = p_ld or _r8(Tk)
        probs = Flat((B, H, Tq, p_ld), torch.float32 if probs_dtype != _lib.BF16 else torch.bfloat16)
        kw = _base_args(K, B, H, Tq, Tk, _lib.BF16, qb, kb, vb, out, False, maxpos, pe_dev, None, 0.0, p_ld)
        a = K.attn_args(**kw, probs=probs.ptr if probs_dtype is not None else None,
                        probs_dtype=probs_dtype if probs_dtype is not None else 0)
        return a, out, probs, (qb, kb, vb, pe_dev)

    def untouched(*bufs):
        torch.cuda.synchronize()
        for b in bufs:
            assert bool(torch.isnan(b.flat.float()).all()), "rejected call wrote its output"

    a, out, probs, keep = fused_args(1, 2, 64, 321)
    with pytest.raises(RuntimeError, match="st5_attn_fused_fwd"):
        K.attn_fused_fwd(a, None)
    untouched(out)
    a, out, probs, keep = fused_args(1, 2, 65, 65, maxpos=64)
    with pytest.raises(RuntimeError, match="relative positions"):
        K.attn_fused_fwd(a, None)
    untouched(out)
    a, out, probs, keep = fused_args(1, 2, 100, 313, p_ld=316)
    psave = Flat((1, 2, 100, 316), torch.bfloat16)
    inv_l = Flat((1, 2, 100), torch.float32)
    with pytest.raises(RuntimeError, match="psave"):
        K.attn_flash_fwd(a, None, psave.ptr, inv_l.ptr)
    untouched(out, psave, inv_l)
    a, out, probs, keep = fused_args(1, 2, 64, 200, probs_dtype=_lib.BF16)
    with pytest.raises(RuntimeError, match="fp32"):
        K.attn_flash_fwd(a, None)
    untouched(out, probs)
    s = Flat((1, 1, 4, 520), torch.float32, fill=0.0)
    P = Flat((1, 1, 4, 520), torch.bfloat16)
    with pytest.raises(RuntimeError, match="st5_attn_softmax_fwd"):
        K.attn_softmax_fwd(s.ptr, None, None, P.ptr, None, None, 1, 1, 4, 513, 520, False, 0, 0.0, 0, 0)
    untouched(P)
