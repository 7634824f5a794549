"""Raw (non-autograd) Python wrappers over the C ABI. Tensors are torch CUDA tensors used purely as device buffers;
every call goes to libspeecht5_b200.so on the current CUDA stream. No fallbacks."""
import ctypes as C

import torch

from . import _lib
from ._lib import ACT_IDS, BF16, F32, AttnArgs, GemmArgs


LAUNCHES = 0      # kernels of libspeecht5_b200.so launched through this module (bench.py reports it)
GEMM_RECORD = None  # when a list: every st5_gemm_bf16 argument block is appended (bench.py roofline replay)


def _count(n):
    global LAUNCHES
    LAUNCHES += n


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def dtype_id(t):
    if t.dtype == torch.float32:
        return F32
    if t.dtype == torch.bfloat16:
        return BF16
    raise TypeError(f"unsupported activation dtype {t.dtype}")


def _require_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise RuntimeError("speecht5_b200 kernels need CUDA tensors (no CPU fallback)")


def gemm(a, b, out, *, M, N, K, a_mn=False, b_mn=False, a_ld=None, b_ld=None, c_ld=None, nb1=1, nb2=1,
         a_bs=(0, 0), b_bs=(0, 0), c_bs=(0, 0), bias=None, bias2=None, bias2_rows=0, residual=None, c_pre=None,
         act=None, alpha=1.0, accumulate=False, drop_p=0.0, seed=0, offset=0, actgrad_pre=None, actgrad_act=None):
    """out[z][m][n] = epi(alpha * sum_k A[z][m][k] B[z][n][k]); see st5_gemm_bf16 in include/speecht5_b200.h."""
    _require_cuda(a, b, out)
    assert a.dtype == torch.bfloat16 and b.dtype == torch.bfloat16
    g = GemmArgs()
    g.M, g.N, g.K, g.nb1, g.nb2 = M, N, K, nb1, nb2
    g.a_mn, g.b_mn = int(a_mn), int(b_mn)
    g.c_fp32 = 1 if out.dtype == torch.float32 else 0
    g.act = ACT_IDS[act]
    g.accumulate = int(accumulate)
    g.bias2_rows = bias2_rows
    g.a, g.a_ld, g.a_bs1, g.a_bs2 = a.data_ptr(), (a_ld if a_ld is not None else (M if a_mn else K)), a_bs[0], a_bs[1]
    g.b, g.b_ld, g.b_bs1, g.b_bs2 = b.data_ptr(), (b_ld if b_ld is not None else (N if b_mn else K)), b_bs[0], b_bs[1]
    g.c, g.c_ld, g.c_bs1, g.c_bs2 = out.data_ptr(), (c_ld if c_ld is not None else N), c_bs[0], c_bs[1]
    g.c_pre = None if c_pre is None else c_pre.data_ptr()
    g.bias = None if bias is None else bias.data_ptr()
    g.bias2 = None if bias2 is None else bias2.data_ptr()
    g.residual = None if residual is None else residual.data_ptr()
    if bias is not None:
        assert bias.dtype == torch.float32
    if bias2 is not None:
        assert bias2.dtype == torch.float32
    if residual is not None:
        assert residual.dtype == out.dtype
    if c_pre is not None:
        assert c_pre.dtype == out.dtype
    g.alpha = alpha
    g.drop_p, g.drop_seed, g.drop_offset = drop_p, seed, offset
    if actgrad_pre is not None:
        assert actgrad_pre.dtype == out.dtype
        g.actgrad_pre, g.actgrad_act = actgrad_pre.data_ptr(), ACT_IDS[actgrad_act]
    lib = _lib.load()
    _lib.check(lib.st5_gemm_bf16(C.byref(g), _stream()), "st5_gemm_bf16")
    _count(1)
    if GEMM_RECORD is not None:
        g._keep = (a, b, out, c_pre, bias, bias2, residual, actgrad_pre)  # keep the operands alive for the replay
        GEMM_RECORD.append(g)
    return out


def gemm_replay(records):
    """Re-issue recorded GEMM launches back to back on the current stream (timing only)."""
    lib = _lib.load()
    st = _stream()
    for g in records:
        _lib.check(lib.st5_gemm_bf16(C.byref(g), st), "st5_gemm_bf16")


def cast_bf16(src, hi, lo=None):
    """2-D strided fp32 -> bf16 (hi) and optional bf16 residual (lo)."""
    _require_cuda(src, hi)
    assert src.dtype == torch.float32 and src.dim() == 2 and src.stride(1) == 1
    rows, cols = src.shape
    assert hi.stride(1) == 1 and (lo is None or lo.stride() == hi.stride())
    lib = _lib.load()
    _lib.check(lib.st5_cast_bf16(_ptr(src), src.stride(0), _ptr(hi), _ptr(lo), hi.stride(0), rows, cols, _stream()),
               "st5_cast_bf16")
    _count(1)


def posenc_fwd(tokens, emb, x, pe, alpha, y, drop_p=0.0, seed=0, offset=0):
    B, T, Cc = y.shape
    lib = _lib.load()
    _lib.check(lib.st5_posenc_fwd(_ptr(tokens), _ptr(emb), _ptr(x), _ptr(pe), _ptr(alpha), _ptr(y), dtype_id(y), B, T,
                                  Cc, drop_p, seed, offset, _stream()), "st5_posenc_fwd")
    _count(1)


def posenc_bwd(dy, tokens, padding_idx, pe, dx, demb, dalpha, drop_p=0.0, seed=0, offset=0):
    B, T, Cc = dy.shape
    lib = _lib.load()
    _lib.check(lib.st5_posenc_bwd(_ptr(dy), _ptr(tokens), padding_idx, _ptr(pe), _ptr(dx), _ptr(demb), _ptr(dalpha),
                                  dtype_id(dy), B, T, Cc, drop_p, seed, offset, _stream()), "st5_posenc_bwd")
    _count(1)


def ln_fwd(x, residual, gamma, beta, y, s_out, mean, rstd, eps, drop_p=0.0, seed=0, offset=0, residual_f32=None,
           y_f32=None):
    Cc = x.shape[-1]
    rows = x.numel() // Cc
    lib = _lib.load()
    if residual_f32 is not None or y_f32 is not None:
        assert (residual_f32 is None or residual_f32.dtype == torch.float32) and (y_f32 is None or y_f32.dtype == torch.float32)
        _lib.check(lib.st5_ln_fwd_stream(_ptr(x), _ptr(residual), _ptr(residual_f32), _ptr(gamma), _ptr(beta), _ptr(y),
                                         _ptr(y_f32), _ptr(s_out), _ptr(mean), _ptr(rstd), dtype_id(x), rows, Cc, eps,
                                         drop_p, seed, offset, _stream()), "st5_ln_fwd_stream")
    else:
        _lib.check(lib.st5_ln_fwd(_ptr(x), _ptr(residual), _ptr(gamma), _ptr(beta), _ptr(y), _ptr(s_out), _ptr(mean),
                                  _ptr(rstd), dtype_id(x), rows, Cc, eps, drop_p, seed, offset, _stream()), "st5_ln_fwd")
    _count(1)


def ln_fwd_wide(x, residual, gamma, beta, y, mean=None, rstd=None, eps=1e-5):
    """st5_ln_fwd_wide: y = LayerNorm(x + residual) for rows of 8 <= C <= 2048 channels, forward only (no dropout)."""
    _require_cuda(x, residual, gamma, beta, y, mean, rstd)
    Cc = x.shape[-1]
    rows = x.numel() // Cc
    _lib.check(_lib.load().st5_ln_fwd_wide(_ptr(x), _ptr(residual), _ptr(gamma), _ptr(beta), _ptr(y), _ptr(mean),
                                           _ptr(rstd), dtype_id(x), rows, Cc, eps, _stream()), "st5_ln_fwd_wide")
    _count(1)


def ln_bwd(dy, s, mean, rstd, gamma, ds, dx, dgamma, dbeta, drop_p=0.0, seed=0, offset=0, dxsum=None):
    """dxsum (optional, fp32 [C], accumulated): column sums of dx = the bias gradient of the projection that fed x."""
    Cc = dy.shape[-1]
    rows = dy.numel() // Cc
    lib = _lib.load()
    if dxsum is not None:
        assert dxsum.dtype == torch.float32 and dxsum.numel() >= Cc and dxsum.is_contiguous()
    _lib.check(lib.st5_ln_bwd(_ptr(dy), _ptr(s), _ptr(mean), _ptr(rstd), _ptr(gamma), _ptr(ds), _ptr(dx),
                              _ptr(dgamma), _ptr(dbeta), _ptr(dxsum), dtype_id(dy), rows, Cc, drop_p, seed, offset,
                              _stream()), "st5_ln_bwd")
    fused = (dgamma is not None or dbeta is not None or dxsum is not None) and (rows >= 64 or dxsum is not None)
    _count(1 if fused or (dgamma is None and dbeta is None) else 2)


def lrelu_pad(x, out, d, ph, pad, slope):
    """st5_lrelu_pad: out [B, n_in, C] <- leaky_relu(x [B, T, C]) at frames ph + d*m - pad (zeros outside [0, T))."""
    _require_cuda(x, out)
    assert x.dtype == torch.bfloat16 and out.dtype == torch.bfloat16 and x.is_contiguous() and out.is_contiguous()
    B, T, Cc = x.shape
    assert out.shape[0] == B and out.shape[2] == Cc
    _lib.check(_lib.load().st5_lrelu_pad(_ptr(x), _ptr(out), B, T, Cc, out.shape[1], int(d), int(ph), int(pad),
                                         float(slope), _stream()), "st5_lrelu_pad")
    _count(1)


def lrelu_pad_len(x, out, d, ph, pad, slope, lengths, len_mult=1):
    """st5_lrelu_pad_len: lrelu_pad with the source frames of row b limited to [0, clamp(lengths[b] * len_mult, 0, T));
    lengths: int32 [B] device tensor (None: T for every row)."""
    _require_cuda(x, out, lengths)
    assert x.dtype == torch.bfloat16 and out.dtype == torch.bfloat16 and x.is_contiguous() and out.is_contiguous()
    B, T, Cc = x.shape
    assert out.shape[0] == B and out.shape[2] == Cc
    assert lengths is None or (lengths.dtype == torch.int32 and lengths.is_contiguous() and lengths.numel() >= B)
    _lib.check(_lib.load().st5_lrelu_pad_len(_ptr(x), _ptr(out), B, T, Cc, out.shape[1], int(d), int(ph), int(pad),
                                             float(slope), _ptr(lengths), int(len_mult), _stream()),
               "st5_lrelu_pad_len")
    _count(1)


def dropout(x, y, drop_p, seed, offset):
    lib = _lib.load()
    _lib.check(lib.st5_dropout(_ptr(x), _ptr(y), dtype_id(x), x.numel(), drop_p, seed, offset, _stream()),
               "st5_dropout")
    _count(1)


def act_bwd(dy, pre, dpre, act, drop_p=0.0, seed=0, offset=0):
    lib = _lib.load()
    _lib.check(lib.st5_act_bwd(_ptr(dy), _ptr(pre), _ptr(dpre), dtype_id(dy), ACT_IDS[act], dy.numel(), drop_p, seed,
                               offset, _stream()), "st5_act_bwd")
    _count(1)


def colsum(x2d, out, group_rows=0, accumulate=False, ld=None):
    rows, cols = x2d.shape
    lib = _lib.load()
    _lib.check(lib.st5_colsum(_ptr(x2d), ld if ld is not None else x2d.stride(0), _ptr(out), dtype_id(x2d), rows, cols,
                              group_rows, int(accumulate), _stream()), "st5_colsum")
    _count(1)


def attn_args(**kw):
    a = AttnArgs()
    for k, v in kw.items():
        if isinstance(v, torch.Tensor):
            v = v.data_ptr()
        setattr(a, k, v)
    return a


def attn_fwd(a):
    lib = _lib.load()
    _lib.check(lib.st5_attn_fwd(C.byref(a), _stream()), "st5_attn_fwd")
    _count(1)


def _decode_fields(d, B, q, k, v, out, H, scale, key_pad, probs, ws):
    """Fill an AttnDecodeArgs from strided views: q [B, 1, H*hd], k / v [*, Tk, H*hd], out [B, 1, H*hd]."""
    d.B, d.H, d.Tk, d.dtype = B, H, k.shape[1], dtype_id(out)
    d.q, d.q_bs = q.data_ptr(), q.stride(0)
    d.k, d.k_ld, d.k_bs = k.data_ptr(), k.stride(1), k.stride(0)
    d.v, d.v_ld, d.v_bs = v.data_ptr(), v.stride(1), v.stride(0)
    d.key_pad, d.out, d.o_bs, d.probs = _ptr(key_pad), out.data_ptr(), out.stride(0), _ptr(probs)
    d.scale, d.ws = scale, _ptr(ws)


def _decode_ws(nws, out):
    return torch.empty(nws, dtype=torch.float32, device=out.device) if nws > 0 else None


def attn_decode_fwd(q, k, v, out, *, H, scale, key_pad=None, probs=None):
    """st5_attn_decode_fwd (include/speecht5_b200.h): one query row per (utterance, head). q [B, 1, H*64] and
    k / v [B, Tk, H*64] are strided views (e.g. column blocks of a fused projection buffer), out [B, 1, H*64];
    probs (optional) a contiguous fp32 [B, H, 1, Tk] tensor that receives the probabilities."""
    _require_cuda(q, k, v, out, key_pad, probs)
    assert q.dtype == k.dtype == v.dtype == out.dtype and k.stride(2) == 1 and v.stride(2) == 1
    B, Tk = k.shape[0], k.shape[1]
    assert probs is None or (probs.dtype == torch.float32 and probs.is_contiguous() and probs.numel() == B * H * Tk)
    lib = _lib.load()
    nws = lib.st5_attn_decode_ws_floats(B, H, Tk, int(probs is not None))
    a = _lib.AttnDecodeArgs()
    _decode_fields(a, B, q, k, v, out, H, scale, key_pad, probs, _decode_ws(nws, out))
    _lib.check(lib.st5_attn_decode_fwd(C.byref(a), _stream()), "st5_attn_decode_fwd")
    _count(1 if nws == 0 else 2)


def attn_lineage_fwd(q, k, v, out, *, H, scale, key_pad=None, kv_rows=None, kv_div=1):
    """st5_attn_lineage_fwd (include/speecht5_b200.h): attn_decode_fwd for B query rows q [B, 1, H*64] whose key /
    value j lives in batch row kv_rows[b, j] (int32 [B, >= Tk]) of k / v [*, Tk, H*64], or in row b // kv_div."""
    _require_cuda(q, k, v, out, key_pad, kv_rows)
    assert q.dtype == k.dtype == v.dtype == out.dtype and k.stride(2) == 1 and v.stride(2) == 1
    B, Tk = q.shape[0], k.shape[1]
    assert kv_rows is None or (kv_rows.dtype == torch.int32 and kv_rows.stride(1) == 1 and kv_rows.shape[0] == B)
    lib = _lib.load()
    nws = lib.st5_attn_decode_ws_floats(B, H, Tk, 0)
    a = _lib.AttnLineageArgs()
    _decode_fields(a.base, B, q, k, v, out, H, scale, key_pad, None, _decode_ws(nws, out))
    a.kv_rows, a.kv_rows_ld, a.kv_div = _ptr(kv_rows), (kv_rows.stride(0) if kv_rows is not None else 0), kv_div
    _lib.check(lib.st5_attn_lineage_fwd(C.byref(a), _stream()), "st5_attn_lineage_fwd")
    _count(1 if nws == 0 else 2)


def attn_decode_hd_fwd(q, k, v, out, *, H, head_dim, scale, key_pad=None, probs=None):
    """st5_attn_decode_hd_fwd: attn_decode_fwd for heads of `head_dim` (64 or 80) channels, q / out [B, 1, H*head_dim],
    k / v [B, Tk, H*head_dim]."""
    _require_cuda(q, k, v, out, key_pad, probs)
    assert q.dtype == k.dtype == v.dtype == out.dtype and k.stride(2) == 1 and v.stride(2) == 1
    B, Tk = k.shape[0], k.shape[1]
    assert probs is None or (probs.dtype == torch.float32 and probs.is_contiguous() and probs.numel() == B * H * Tk)
    lib = _lib.load()
    nws = lib.st5_attn_decode_hd_ws_floats(B, H, Tk, int(probs is not None), head_dim)
    if nws < 0:
        raise ValueError(f"one-row attention over heads of {head_dim} channels: 64 and 80 are built")
    a = _lib.AttnDecodeArgs()
    _decode_fields(a, B, q, k, v, out, H, scale, key_pad, probs, _decode_ws(nws, out))
    _lib.check(lib.st5_attn_decode_hd_fwd(C.byref(a), head_dim, _stream()), "st5_attn_decode_hd_fwd")
    _count(1 if nws == 0 else 2)


def attn_lineage_hd_fwd(q, k, v, out, *, H, head_dim, scale, key_pad=None, kv_rows=None, kv_div=1):
    """st5_attn_lineage_hd_fwd: attn_lineage_fwd for heads of `head_dim` (64 or 80) channels."""
    _require_cuda(q, k, v, out, key_pad, kv_rows)
    assert q.dtype == k.dtype == v.dtype == out.dtype and k.stride(2) == 1 and v.stride(2) == 1
    B, Tk = q.shape[0], k.shape[1]
    assert kv_rows is None or (kv_rows.dtype == torch.int32 and kv_rows.stride(1) == 1 and kv_rows.shape[0] == B)
    lib = _lib.load()
    nws = lib.st5_attn_decode_hd_ws_floats(B, H, Tk, 0, head_dim)
    if nws < 0:
        raise ValueError(f"one-row attention over heads of {head_dim} channels: 64 and 80 are built")
    a = _lib.AttnLineageArgs()
    _decode_fields(a.base, B, q, k, v, out, H, scale, key_pad, None, _decode_ws(nws, out))
    a.kv_rows, a.kv_rows_ld, a.kv_div = _ptr(kv_rows), (kv_rows.stride(0) if kv_rows is not None else 0), kv_div
    _lib.check(lib.st5_attn_lineage_hd_fwd(C.byref(a), head_dim, _stream()), "st5_attn_lineage_hd_fwd")
    _count(1 if nws == 0 else 2)


def beam_topk(logits, cum, mask, inv_temp, eos, t, min_len, max_len, cand_score, cand_token, cand_beam, *, K,
              lm_logits=None, lm_weight=0.0):
    """st5_beam_topk: logits [B*K, V] (row pitch logits.stride(0), fp32 / bf16), cum [B*K] fp32, mask [V] fp32; t /
    min_len / max_len int64 device scalars; cand_* [B, 2K] (fp32, int32, int32) receive the first min(2K, F-1).
    With lm_logits [B*K, V_lm] (V_lm <= V, fp32 / bf16, row pitch lm_logits.stride(0)): st5_beam_topk_lm, which adds
    lm_weight * log_softmax(lm_logits) to the first V_lm log-probabilities before the masking."""
    _require_cuda(logits, cum, mask, t, min_len, max_len, cand_score, cand_token, cand_beam, lm_logits)
    assert logits.stride(1) == 1 and cum.dtype == torch.float32 and mask.dtype == torch.float32
    assert t.dtype == min_len.dtype == max_len.dtype == torch.int64
    assert cand_score.dtype == torch.float32 and cand_token.dtype == cand_beam.dtype == torch.int32
    BK, V = logits.shape
    B = BK // K
    lib = _lib.load()
    ws = torch.empty(max(1, lib.st5_beam_topk_ws_floats(B, K)), dtype=torch.float32, device=logits.device)
    args = (_ptr(logits), logits.stride(0), dtype_id(logits), B, K, V, _ptr(cum), _ptr(mask), float(inv_temp), int(eos),
            _ptr(t), _ptr(min_len), _ptr(max_len), _ptr(cand_score), _ptr(cand_token), _ptr(cand_beam), _ptr(ws))
    if lm_logits is None:
        _lib.check(lib.st5_beam_topk(*args, _stream()), "st5_beam_topk")
    else:
        assert lm_logits.stride(1) == 1 and lm_logits.shape[0] == BK
        if lm_logits.shape[1] > V:
            raise ValueError(f"the LM vocabulary ({lm_logits.shape[1]}) is larger than the decoder's ({V})")
        _lib.check(lib.st5_beam_topk_lm(*args, _ptr(lm_logits), lm_logits.stride(0), dtype_id(lm_logits),
                                        lm_logits.shape[1], float(lm_weight), _stream()), "st5_beam_topk_lm")
    _count(2)


def beam_update(st, *, K, V, eos, normalize, len_penalty):
    """st5_beam_update on the state dict `st` (speecht5_b200/incremental.BeamGraph.state: the tensors the header names,
    lin / tok / score / fin_tok / fin_pos [.., T] with T = their last dimension)."""
    names = ("t", "max_len", "cand_score", "cand_token", "cand_beam", "lin", "tok", "score", "ignore", "finished",
             "parent", "cur_tok", "cur_score", "fin_n", "fin_tok", "fin_pos", "fin_len", "fin_score", "stop")
    _require_cuda(*(st[n] for n in names))
    B, T = st["finished"].shape[0], st["lin"].shape[-1]
    lib = _lib.load()
    _lib.check(lib.st5_beam_update(B, K, V, T, int(eos), *(_ptr(st[n]) for n in names[:2]), int(bool(normalize)),
                                   float(len_penalty), *(_ptr(st[n]) for n in names[2:]), _stream()), "st5_beam_update")
    _count(2)


def attn_bwd(a):
    lib = _lib.load()
    _lib.check(lib.st5_attn_bwd(C.byref(a), _stream()), "st5_attn_bwd")
    _count(3)


def attn_fused_fwd(a, lse, psave=None, inv_l=None, out_f32=None):
    lib = _lib.load()
    _lib.check(lib.st5_attn_fused_fwd(C.byref(a), _ptr(lse), _ptr(psave), _ptr(inv_l), _ptr(out_f32), _stream()),
               "st5_attn_fused_fwd")
    _count(1)


def attn_flash_fwd(a, lse, psave=None, inv_l=None, out_f32=None):
    lib = _lib.load()
    _lib.check(lib.st5_attn_flash_fwd(C.byref(a), _ptr(lse), _ptr(psave), _ptr(inv_l), _ptr(out_f32), _stream()),
               "st5_attn_flash_fwd")
    _count(1)


def attn_fused_bwd(a, psave, inv_l, out_f32, delta, dq_acc, ext_heads=0):
    lib = _lib.load()
    _lib.check(lib.st5_attn_fused_bwd(C.byref(a), _ptr(psave), _ptr(inv_l), _ptr(out_f32), _ptr(delta), _ptr(dq_acc),
                                      int(ext_heads), _stream()),
               "st5_attn_fused_bwd")
    _count(3 if (a.dprobs_ext and 0 < int(ext_heads) < a.H) else 2)  # (+ the guided heads' row-constant launch)



def attn_softmax_fwd(s, qp, key_pad, p, probs_f32, pdrop, B, H, Tq, Tk, p_ld, causal, maxpos, drop_p, seed, offset):
    lib = _lib.load()
    _lib.check(lib.st5_attn_softmax_fwd(_ptr(s), _ptr(qp), qp.shape[-1] if qp is not None else 0, _ptr(key_pad),
                                        _ptr(p), _ptr(probs_f32), _ptr(pdrop), B, H, Tq, Tk, p_ld, int(causal), maxpos,
                                        drop_p, seed, offset, _stream()), "st5_attn_softmax_fwd")
    _count(1)


def attn_ds(p, dp, dp_ext, ds, pdrop, B, H, Tq, Tk, p_ld, drop_p, seed, offset):
    lib = _lib.load()
    _lib.check(lib.st5_attn_ds(_ptr(p), _ptr(dp), _ptr(dp_ext), _ptr(ds), _ptr(pdrop), B, H, Tq, Tk, p_ld, drop_p, seed,
                               offset, _stream()), "st5_attn_ds")
    _count(1)


def attn_dqp_scatter(ds, dqp, B, H, Tq, Tk, p_ld, maxpos, h_major=False):
    lib = _lib.load()
    _lib.check(lib.st5_attn_dqp_scatter(_ptr(ds), _ptr(dqp), B, H, Tq, Tk, p_ld, maxpos, int(h_major), _stream()),
               "st5_attn_dqp_scatter")
    _count(1)


def bn_fwd(x, x_ld, gamma, beta, running_mean, running_var, save_mean, save_rstd, y, y_ld, y_pre, rows, Cc, training,
           momentum, eps, act, drop_p, seed, offset, scratch):
    lib = _lib.load()
    _lib.check(lib.st5_bn_fwd(_ptr(x), x_ld, _ptr(gamma), _ptr(beta), _ptr(running_mean), _ptr(running_var),
                              _ptr(save_mean), _ptr(save_rstd), _ptr(y), y_ld, _ptr(y_pre), dtype_id(x), rows, Cc,
                              int(training), momentum, eps, ACT_IDS[act], drop_p, seed, offset, _ptr(scratch),
                              _stream()), "st5_bn_fwd")
    _count(5)


def bn_bwd(dy, dy_ld, x, x_ld, y_pre, gamma, save_mean, save_rstd, dx, dx_ld, dgamma, dbeta, rows, Cc, act, drop_p,
           seed, offset, scratch):
    lib = _lib.load()
    _lib.check(lib.st5_bn_bwd(_ptr(dy), dy_ld, _ptr(x), x_ld, _ptr(y_pre), _ptr(gamma), _ptr(save_mean),
                              _ptr(save_rstd), _ptr(dx), dx_ld, _ptr(dgamma), _ptr(dbeta), dtype_id(x), rows, Cc,
                              ACT_IDS[act], drop_p, seed, offset, _ptr(scratch), _stream()), "st5_bn_bwd")
    _count(2)


def conv0_gn_gelu_fwd(wave, w, gamma, beta, y, mean, rstd, stride, eps, act):
    """st5_conv0_gn_gelu_fwd: wave [B, n] fp32, w [C, K] fp32 -> y [B, T0, C] (y.dtype)."""
    _require_cuda(wave, w, y)
    assert wave.dtype == torch.float32 and w.dtype == torch.float32 and wave.is_contiguous() and w.is_contiguous()
    B, n = wave.shape
    Cc, Kt = w.shape
    lib = _lib.load()
    ws = torch.empty(lib.st5_conv0_ws_floats(B, n, Cc, Kt, stride), device=wave.device, dtype=torch.float32)
    _lib.check(lib.st5_conv0_gn_gelu_fwd(_ptr(wave), _ptr(w), _ptr(gamma), _ptr(beta), _ptr(y), dtype_id(y), _ptr(mean),
                                         _ptr(rstd), _ptr(ws), B, n, Cc, Kt, stride, eps, ACT_IDS[act], _stream()),
               "st5_conv0_gn_gelu_fwd")
    _count(3)


def conv0_gn_gelu_bwd(dy, wave, w, gamma, beta, mean, rstd, dw, dgamma, dbeta, stride, act):
    """st5_conv0_gn_gelu_bwd: dw / dgamma / dbeta (fp32) are accumulated."""
    _require_cuda(dy, wave, w)
    assert dy.is_contiguous()
    B, n = wave.shape
    Cc, Kt = w.shape
    lib = _lib.load()
    ws = torch.empty(lib.st5_conv0_ws_floats(B, n, Cc, Kt, stride), device=wave.device, dtype=torch.float32)
    _lib.check(lib.st5_conv0_gn_gelu_bwd(_ptr(dy), _ptr(wave), _ptr(w), _ptr(gamma), _ptr(beta), _ptr(mean), _ptr(rstd),
                                         _ptr(dw), _ptr(dgamma), _ptr(dbeta), _ptr(ws), dtype_id(dy), B, n, Cc, Kt,
                                         stride, ACT_IDS[act], _stream()), "st5_conv0_gn_gelu_bwd")
    _count(4)


def conv0_ln_gelu_fwd(wave, w, gamma, beta, y, mean, rstd, stride, eps, act):
    """st5_conv0_ln_gelu_fwd: wave [B, n] fp32, w [C, K] fp32 -> y [B, T0, C] (y.dtype), mean / rstd [B * T0]."""
    _require_cuda(wave, w, y)
    assert wave.dtype == torch.float32 and w.dtype == torch.float32 and wave.is_contiguous() and w.is_contiguous()
    B, n = wave.shape
    Cc, Kt = w.shape
    lib = _lib.load()
    _lib.check(lib.st5_conv0_ln_gelu_fwd(_ptr(wave), _ptr(w), _ptr(gamma), _ptr(beta), _ptr(y), dtype_id(y), _ptr(mean),
                                         _ptr(rstd), B, n, Cc, Kt, stride, eps, ACT_IDS[act], _stream()),
               "st5_conv0_ln_gelu_fwd")
    _count(1)


def conv0_ln_gelu_bwd(dy, wave, w, gamma, beta, mean, rstd, dw, dgamma, dbeta, stride, act):
    """st5_conv0_ln_gelu_bwd: dw / dgamma / dbeta (fp32) are accumulated."""
    _require_cuda(dy, wave, w)
    assert dy.is_contiguous()
    B, n = wave.shape
    Cc, Kt = w.shape
    lib = _lib.load()
    ws = torch.empty(lib.st5_conv0_ln_ws_floats(B, n, Cc, Kt, stride), device=wave.device, dtype=torch.float32)
    _lib.check(lib.st5_conv0_ln_gelu_bwd(_ptr(dy), _ptr(wave), _ptr(w), _ptr(gamma), _ptr(beta), _ptr(mean), _ptr(rstd),
                                         _ptr(dw), _ptr(dgamma), _ptr(dbeta), _ptr(ws), dtype_id(dy), B, n, Cc, Kt,
                                         stride, ACT_IDS[act], _stream()), "st5_conv0_ln_gelu_bwd")
    _count(4)


def act_fwd(x, y, act):
    """st5_act_fwd: y = act(x), contiguous tensors of one dtype."""
    _require_cuda(x, y)
    assert x.is_contiguous() and y.is_contiguous() and x.dtype == y.dtype
    lib = _lib.load()
    _lib.check(lib.st5_act_fwd(_ptr(x), _ptr(y), dtype_id(x), ACT_IDS[act], x.numel(), _stream()), "st5_act_fwd")
    _count(1)


def ctc_loss(logits, targets, tgt_offsets, input_lengths, target_lengths, nll, grad, s_max, blank, zero_infinity):
    """logits [T, B, V] fp32 (inner stride 1); see st5_ctc_loss (rows + concurrent alpha / beta sweeps + gradient rows)."""
    _require_cuda(logits, targets, nll)
    assert logits.dtype == torch.float32 and logits.stride(2) == 1
    for t in (targets, tgt_offsets, input_lengths, target_lengths):
        assert t.dtype == torch.int64 and t.is_contiguous()
    T, B, V = logits.shape
    assert grad is None or (grad.dtype == torch.float32 and grad.stride() == logits.stride())
    lib = _lib.load()
    ws = torch.empty(lib.st5_ctc_ws_floats(T, B, s_max), device=logits.device, dtype=torch.float32)
    _lib.check(lib.st5_ctc_loss(_ptr(logits), logits.stride(0), logits.stride(1), _ptr(targets), _ptr(tgt_offsets),
                                _ptr(input_lengths), _ptr(target_lengths), _ptr(nll), _ptr(grad), _ptr(ws), T, B, V,
                                s_max, blank, int(zero_infinity), _stream()), "st5_ctc_loss")
    _count(3 if grad is not None else 2)


def tts_loss_ws_floats(B, L):
    return int(_lib.load().st5_tts_loss_ws_floats(B, L))


def guided_attn_ws_floats(n_layers, B, heads, T_out):
    return int(_lib.load().st5_guided_attn_ws_floats(n_layers, B, heads, T_out))


def tts_loss_fwd(after, before, logits, ys, labels, olens, r, pos_weight, sums, out):
    """st5_tts_loss_fwd: out[0..2] = l1, l2, bce of Tacotron2Loss (masked means); after / before [B, L, D] fp32."""
    _require_cuda(after, before, logits, ys, labels, olens, sums, out)
    B, L, D = after.shape
    for t in (after, before, logits):
        assert t.dtype == torch.float32 and t.is_contiguous()
    assert ys.dtype == torch.float32 and ys.stride(2) == 1 and ys.stride(1) == D and ys.shape[1] >= L
    assert labels.dtype == torch.float32 and labels.stride(1) == 1 and olens.dtype == torch.int64 and olens.is_contiguous()
    _lib.check(_lib.load().st5_tts_loss_fwd(_ptr(after), _ptr(before), _ptr(logits), _ptr(ys), ys.stride(0), _ptr(labels),
                                            labels.stride(0), _ptr(olens), B, L, D, r, pos_weight, _ptr(sums), _ptr(out),
                                            _stream()), "st5_tts_loss_fwd")
    _count(2)


def tts_loss_bwd(after, before, logits, ys, labels, olens, sums, g, r, pos_weight, d_after, d_before, d_logits):
    _require_cuda(after, g, d_after)
    B, L, D = after.shape
    assert g.dtype == torch.float32 and g.is_contiguous() and g.numel() == 3
    for t in (d_after, d_before, d_logits):
        assert t.dtype == torch.float32 and t.is_contiguous()
    _lib.check(_lib.load().st5_tts_loss_bwd(_ptr(after), _ptr(before), _ptr(logits), _ptr(ys), ys.stride(0), _ptr(labels),
                                            labels.stride(0), _ptr(olens), _ptr(sums), _ptr(g), B, L, D, r, pos_weight,
                                            _ptr(d_after), _ptr(d_before), _ptr(d_logits), _stream()), "st5_tts_loss_bwd")
    _count(1)


def _att_layout(atts):
    B, H, T_out, T_in = atts[0].shape
    p_ld = atts[0].stride(2)
    for a in atts:
        assert a.dtype == torch.float32 and a.shape == atts[0].shape and a.stride(3) == 1 and a.stride(2) == p_ld
        assert a.stride(1) == T_out * p_ld and a.stride(0) == H * T_out * p_ld, "attention probabilities: [B,H,T_out,p_ld] pitch"
    ptrs = (C.c_void_p * len(atts))(*[a.data_ptr() for a in atts])
    return B, H, T_out, T_in, p_ld, ptrs


def guided_attn_fwd(atts, heads, ilens, olens, r, sigma, alpha, gsum, out):
    """st5_guided_attn_fwd over the first `heads` heads of each tensor in `atts` ([B, H, T_out, T_in] fp32 views)."""
    _require_cuda(atts[0], ilens, olens, gsum, out)
    B, H, T_out, T_in, p_ld, ptrs = _att_layout(atts)
    assert ilens.dtype == torch.int64 and olens.dtype == torch.int64 and ilens.is_contiguous() and olens.is_contiguous()
    _lib.check(_lib.load().st5_guided_attn_fwd(ptrs, len(atts), B, H, heads, T_out, T_in, p_ld, _ptr(ilens), _ptr(olens),
                                               r, sigma, alpha, _ptr(gsum), _ptr(out), _stream()), "st5_guided_attn_fwd")
    _count(2)


def guided_attn_bwd(datts, heads, T_in, ilens, olens, r, sigma, alpha, gsum, g, zero_rest):
    """datts: [B, H, T_out, p_ld] fp32 contiguous buffers (p_ld >= T_in)."""
    _require_cuda(datts[0], gsum, g)
    B, H, T_out, p_ld = datts[0].shape
    for d in datts:
        assert d.dtype == torch.float32 and d.is_contiguous() and d.shape == datts[0].shape
    ptrs = (C.c_void_p * len(datts))(*[d.data_ptr() for d in datts])
    _lib.check(_lib.load().st5_guided_attn_bwd(ptrs, len(datts), B, H, heads, T_out, T_in, p_ld, _ptr(ilens), _ptr(olens),
                                               r, sigma, alpha, _ptr(gsum), _ptr(g), int(zero_rest), _stream()),
               "st5_guided_attn_bwd")
    _count(1)


def l2norm_rows_fwd(x, y, nrm):
    """st5_l2norm_rows_fwd: y [rows, E] fp32 = F.normalize(x, dim=1); nrm [rows] = row norms. x: 2-D, unit inner stride."""
    _require_cuda(x, y, nrm)
    rows, E = x.shape
    assert x.stride(1) == 1 and y.dtype == torch.float32 and y.is_contiguous() and y.shape == (rows, E)
    _lib.check(_lib.load().st5_l2norm_rows_fwd(_ptr(x), x.stride(0), dtype_id(x), _ptr(y), _ptr(nrm), rows, E,
                                               _stream()), "st5_l2norm_rows_fwd")
    _count(1)


def l2norm_rows_bwd(dy, y, nrm, dx, accumulate=False):
    """st5_l2norm_rows_bwd: dx (2-D, unit inner stride; fp32 when accumulate) <- (or +=) the input gradient."""
    _require_cuda(dy, y, nrm, dx)
    rows, E = y.shape
    assert dy.dtype == torch.float32 and dy.is_contiguous() and dx.stride(1) == 1 and dx.shape == (rows, E)
    _lib.check(_lib.load().st5_l2norm_rows_bwd(_ptr(dy), _ptr(y), _ptr(nrm), _ptr(dx), dx.stride(0), dtype_id(dx),
                                               int(accumulate), rows, E, _stream()), "st5_l2norm_rows_bwd")
    _count(1)


def _margin_args(margin):
    """margin: None or (mode, scale, m, easy_margin)."""
    return (_lib.MARGIN_NONE, 1.0, 0.0, 0) if margin is None else (int(margin[0]), float(margin[1]),
                                                                  float(margin[2]), int(margin[3]))


def margin_ce_fwd(x, mtarget, margin, z_out=None, target=None, eps=0.0, ignore_index=-100, stats=None, lse=None):
    """st5_margin_ce_fwd over x [B, N] fp32 (unit inner stride): margin logits into z_out and / or per-row (loss, nll,
    correct, valid) into stats [B, 4] with lse [B] for the backward."""
    _require_cuda(x, z_out, target, stats, lse)
    B, N = x.shape
    assert x.dtype == torch.float32 and x.stride(1) == 1
    for t in (mtarget, target):
        assert t is None or (t.dtype == torch.int64 and t.is_contiguous() and t.numel() == B)
    assert z_out is None or (z_out.dtype == torch.float32 and z_out.stride(1) == 1)
    mode, s, m, easy = _margin_args(margin)
    _lib.check(_lib.load().st5_margin_ce_fwd(_ptr(x), x.stride(0), B, N, _ptr(mtarget), mode, s, m, easy, _ptr(z_out),
                                             z_out.stride(0) if z_out is not None else 0, _ptr(target), eps,
                                             ignore_index, _ptr(stats), _ptr(lse), _stream()), "st5_margin_ce_fwd")
    _count(1)


def margin_ce_bwd(x, mtarget, margin, dx, target=None, eps=0.0, ignore_index=-100, lse=None, gstat=None, dz=None):
    """st5_margin_ce_bwd: dx [B, N] fp32 = d logits from the loss (target, lse, gstat [2] device floats) or from dz."""
    _require_cuda(x, dx, dz)
    B, N = x.shape
    assert dx.dtype == torch.float32 and dx.stride(1) == 1
    assert gstat is None or (gstat.dtype == torch.float32 and gstat.is_contiguous())
    assert dz is None or (dz.dtype == torch.float32 and dz.stride(1) == 1)
    mode, s, m, easy = _margin_args(margin)
    _lib.check(_lib.load().st5_margin_ce_bwd(_ptr(x), x.stride(0), B, N, _ptr(mtarget), mode, s, m, easy, _ptr(target),
                                             eps, ignore_index, _ptr(lse), _ptr(gstat), _ptr(dz),
                                             dz.stride(0) if dz is not None else 0, _ptr(dx), dx.stride(0), _stream()),
               "st5_margin_ce_bwd")
    _count(1)


def time_mean_fwd(x, y):
    """st5_time_mean_fwd: y [B, C] = x [B, T, C].mean(1) (contiguous, one dtype)."""
    _require_cuda(x, y)
    B, T, Cc = x.shape
    assert x.is_contiguous() and y.is_contiguous() and x.dtype == y.dtype and y.shape == (B, Cc)
    _lib.check(_lib.load().st5_time_mean_fwd(_ptr(x), _ptr(y), dtype_id(x), B, T, Cc, _stream()), "st5_time_mean_fwd")
    _count(1)


def time_mean_bwd(dy, dx):
    _require_cuda(dy, dx)
    B, T, Cc = dx.shape
    assert dy.is_contiguous() and dx.is_contiguous() and dy.dtype == dx.dtype
    _lib.check(_lib.load().st5_time_mean_bwd(_ptr(dy), _ptr(dx), dtype_id(dx), B, T, Cc, _stream()), "st5_time_mean_bwd")
    _count(1)


def sumsq(x, out):
    lib = _lib.load()
    _lib.check(lib.st5_sumsq(_ptr(x), x.numel(), _ptr(out), _stream()), "st5_sumsq")
    _count(1)


def adam_step(p, g, m, v, p_bf16, lr, beta1, beta2, eps, weight_decay, step, grad_norm_sq, max_norm, grad_mul,
              lr_dev=None, step_dev=None):
    lib = _lib.load()
    _lib.check(lib.st5_adam_step(_ptr(p), _ptr(g), _ptr(m), _ptr(v), _ptr(p_bf16), p.numel(), lr, beta1, beta2, eps,
                                 weight_decay, step, _ptr(grad_norm_sq), max_norm, grad_mul, _ptr(lr_dev),
                                 _ptr(step_dev), _stream()), "st5_adam_step")
    _count(1)
