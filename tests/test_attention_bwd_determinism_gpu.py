"""-m gpu: st5_attn_fused_bwd is deterministic. Its dQ is a running fp32 sum over the key blocks in a fixed order, split
between two warpgroups and a prefetching warp, and dK / dV / dS are written once per element; two calls on identical
inputs (fresh NaN scratch each time) must give bit-identical dq, dk, dv and ds. The shapes cover even and odd numbers
of 64-key blocks (Tk = 64, 128, 160, 313), causal masks with Tk > Tq, Tq off a multiple of 64, an external gradient
on the first two heads' probabilities and the relative-position path. Buffers and arguments are laid out as in
tests/test_attention_contract_gpu.py, which checks the values themselves."""
import pytest
import torch

import attention_ref as R
from test_attention_contract_gpu import SCALE, Flat, Rows, _base_args, _key_pad, _layout

pytestmark = pytest.mark.gpu

CASES = [
    dict(entry="fused", B=2, H=2, Tq=64, Tk=64),
    dict(entry="fused", B=3, H=2, Tq=100, Tk=128, pad=True, drop=0.2),
    dict(entry="fused", B=2, H=3, Tq=160, Tk=160, maxpos=160, probe=True, drop=0.1),
    dict(entry="fused", B=2, H=3, Tq=313, Tk=313, causal=True, drop=0.1),
    dict(entry="fused", B=2, H=3, Tq=313, Tk=160, pad=True, drop=0.1, ext_heads=2),
    dict(entry="flash", B=2, H=2, Tq=70, Tk=313, causal=True),
    dict(entry="flash", B=2, H=2, Tq=130, Tk=313, causal=True, drop=0.2),
]


def _id(c):
    return "-".join(f"{k}{v}" for k, v in c.items() if k not in ("B", "H"))


@pytest.mark.parametrize("case", CASES, ids=_id)
def test_fused_bwd_is_bit_identical_across_calls(case):
    from speecht5_b200 import _lib
    from speecht5_b200 import kernels as K
    c = dict(case)
    entry, B, H, Tq, Tk = c.pop("entry"), c.pop("B"), c.pop("H"), c.pop("Tq"), c.pop("Tk")
    causal, maxpos, drop = c.get("causal", False), c.get("maxpos", 0), c.get("drop", 0.0)
    ext_heads = c.get("ext_heads")
    q, k, v, pe = R.make_inputs(B, H, Tq, Tk, seed=5, maxpos=maxpos, probe=c.get("probe", False))
    pe_dev = pe.to(torch.bfloat16).cuda() if pe is not None else None
    kp = _key_pad(c.get("pad", False), B, Tk)
    kp_dev = kp.to(torch.uint8).cuda() if kp is not None else None
    p_ld = (Tk + 7) // 8 * 8
    d = H * 64
    qb, kb, vb = _layout(B, H, Tq, Tk, torch.bfloat16)
    for buf, x in ((qb, q), (kb, k), (vb, v)):
        buf.set(x.cuda())
    out = Rows(B, Tq, H, torch.bfloat16, ld=d + 16, gap=2)
    psave, inv_l = Flat((B, H, Tq, p_ld), torch.bfloat16), Flat((B, H, Tq), torch.float32)
    o32, lse = Flat((B, Tq, d), torch.float32), Flat((B, H, Tq), torch.float32)
    probs = Flat((B, H, Tq, p_ld), torch.float32) if ext_heads is not None else None
    kw = _base_args(K, B, H, Tq, Tk, _lib.BF16, qb, kb, vb, out, causal, maxpos, pe_dev, kp_dev, drop, p_ld)
    assert kw["scale"] == SCALE
    a = K.attn_args(**kw, probs=probs.ptr if probs is not None else None, probs_dtype=_lib.F32)
    fwd = K.attn_flash_fwd if entry == "flash" else K.attn_fused_fwd
    fwd(a, lse.ptr, psave.ptr, inv_l.ptr, o32.ptr)

    gen = torch.Generator().manual_seed(11)
    dout = Rows(B, Tq, H, torch.bfloat16, ld=out.ld, gap=2)
    dout.set(torch.randn(B, H, Tq, 64, generator=gen).to(torch.bfloat16).cuda())
    dpx = None
    if ext_heads is not None:
        dpx = Flat((B, H, Tq, p_ld), torch.float32)
        dpx.t[:, :ext_heads, :, :Tk] = (torch.randn(B, ext_heads, Tq, Tk, generator=gen) * 4.0).cuda()

    def backward():
        dq, dk, dv = (Rows(x.B, x.T, x.H, torch.bfloat16, ld=x.ld, col0=x.col0) for x in (qb, kb, vb))
        delta, dq_acc = Flat((B, H, Tq), torch.float32), Flat((B, Tq, d), torch.float32)
        ds = Flat((B, H, Tq, p_ld), torch.bfloat16) if pe_dev is not None else None
        ab = K.attn_args(**kw, probs=probs.ptr if probs is not None else None, probs_dtype=_lib.F32, dout=dout.ptr,
                         dprobs_ext=dpx.ptr if dpx is not None else None, ds=ds.ptr if ds is not None else None,
                         dq=dq.ptr, dk=dk.ptr, dv=dv.ptr)
        K.attn_fused_bwd(ab, psave.ptr, inv_l.ptr, o32.ptr, delta.ptr, dq_acc.ptr, ext_heads=ext_heads or 0)
        torch.cuda.synchronize()
        res = {"dq": dq.get(), "dk": dk.get(), "dv": dv.get()}
        if ds is not None:
            res["ds"] = ds.get()[..., :Tk]
        return res

    first, second = backward(), backward()
    for name, x in first.items():
        assert not bool(torch.isnan(x.float()).any()), f"{name}: NaN in the result"
        same = x.view(torch.int16) == second[name].view(torch.int16)
        assert bool(same.all()), f"{name}: {int((~same).sum())} elements differ between two identical calls"
