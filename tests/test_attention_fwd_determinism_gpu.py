"""-m gpu: the attention forward is deterministic. Each of its two warpgroups sums its rows over a quad of lanes in a
fixed order, and every output element is written once; two calls on identical inputs (fresh NaN buffers each time)
must give bit-identical out, out_f32, psave, inv_l, lse and probs. The shapes cover even and odd numbers of 64-row
query tiles (a CTA takes two), a lone last tile, causal masks with Tk > Tq, ragged key padding, dropout, returned
probabilities on some heads, relative positions at T = 160 and clipped relative positions at T = 499. Buffers and
arguments are laid out as in tests/test_attention_contract_gpu.py, which checks the values themselves."""
import pytest
import torch

import attention_ref as R
from test_attention_contract_gpu import Flat, Rows, _base_args, _key_pad, _layout

pytestmark = pytest.mark.gpu

CASES = [
    dict(entry="fused", B=2, H=2, Tq=128, Tk=128, drop=0.1),
    dict(entry="fused", B=3, H=2, Tq=192, Tk=100, pad=True, drop=0.2),
    dict(entry="fused", B=2, H=3, Tq=160, Tk=160, maxpos=160, drop=0.1),
    dict(entry="fused", B=2, H=3, Tq=313, Tk=313, causal=True, drop=0.1),
    dict(entry="fused", B=2, H=3, Tq=313, Tk=160, pad=True, drop=0.1, probs_heads=2),
    dict(entry="flash", B=2, H=2, Tq=70, Tk=313, causal=True, drop=0.2, probs_heads=2),
    dict(entry="flash", B=1, H=2, Tq=499, Tk=499, maxpos=160, drop=0.1),
]


def _id(c):
    return "-".join(f"{k}{v}" for k, v in c.items() if k not in ("B", "H"))


@pytest.mark.parametrize("case", CASES, ids=_id)
def test_attention_fwd_is_bit_identical_across_calls(case):
    from speecht5_b200 import _lib
    from speecht5_b200 import kernels as K
    c = dict(case)
    entry, B, H, Tq, Tk = c.pop("entry"), c.pop("B"), c.pop("H"), c.pop("Tq"), c.pop("Tk")
    causal, maxpos, drop = c.get("causal", False), c.get("maxpos", 0), c.get("drop", 0.0)
    probs_heads = c.get("probs_heads")
    q, k, v, pe = R.make_inputs(B, H, Tq, Tk, seed=7, maxpos=maxpos)
    pe_dev = pe.to(torch.bfloat16).cuda() if pe is not None else None
    kp = _key_pad(c.get("pad", False), B, Tk)
    kp_dev = kp.to(torch.uint8).cuda() if kp is not None else None
    p_ld = (Tk + 7) // 8 * 8
    d = H * 64
    qb, kb, vb = _layout(B, H, Tq, Tk, torch.bfloat16)
    for buf, x in ((qb, q), (kb, k), (vb, v)):
        buf.set(x.cuda())
    fwd = K.attn_flash_fwd if entry == "flash" else K.attn_fused_fwd

    def forward():
        out = Rows(B, Tq, H, torch.bfloat16, ld=d + 16, gap=2)
        psave, inv_l = Flat((B, H, Tq, p_ld), torch.bfloat16), Flat((B, H, Tq), torch.float32)
        o32, lse = Flat((B, Tq, d), torch.float32), Flat((B, H, Tq), torch.float32)
        probs = Flat((B, H, Tq, p_ld), torch.float32) if probs_heads is not None else None
        kw = _base_args(K, B, H, Tq, Tk, _lib.BF16, qb, kb, vb, out, causal, maxpos, pe_dev, kp_dev, drop, p_ld)
        a = K.attn_args(**kw, probs=probs.ptr if probs is not None else None, probs_dtype=_lib.F32,
                        probs_heads=probs_heads or 0)
        fwd(a, lse.ptr, psave.ptr, inv_l.ptr, o32.ptr)
        torch.cuda.synchronize()
        res = {"out": out.get(), "out_f32": o32.get(), "psave": psave.get()[..., :Tk], "inv_l": inv_l.get(),
               "lse": lse.get()}
        if probs is not None:
            res["probs"] = probs.get()[:, :probs_heads, :, :Tk]
        return res

    first, second = forward(), forward()
    for name, x in first.items():
        if name != "psave":  # (a causal row's psave is left unwritten right of its last key block)
            assert not bool(torch.isnan(x.float()).any()), f"{name}: NaN in the result"
        view = torch.int16 if x.dtype == torch.bfloat16 else torch.int32
        same = x.contiguous().view(view) == second[name].contiguous().view(view)
        assert bool(same.all()), f"{name}: {int((~same).sum())} elements differ between two identical calls"
