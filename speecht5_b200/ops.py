"""Autograd-visible operators of the SpeechT5 hot path. PyTorch autograd is used only as the tape; every forward and
backward computation below is a call into the hand-written CUDA library (speecht5_b200.kernels -> C ABI).

Two numeric modes (Runtime.dtype):
  * torch.bfloat16 -- throughput mode: bf16 activations, bf16 tensor-core GEMMs with fp32 accumulation, fp32 statistics.
  * torch.float32  -- parity mode: fp32 activations; each GEMM is evaluated as hi*hi + hi*lo + lo*hi over bf16 splits of
    both operands (three accumulate passes of the same wgmma kernel), i.e. ~2^-16 relative operand error.
"""
import os

import torch

from . import kernels as K


class Runtime:
    """Process-wide numeric mode, dropout counter stream and bf16 weight-shadow cache."""

    SEED_PTR_FLAG = 1 << 63

    def __init__(self):
        self.dtype = torch.bfloat16
        self._seed = 1
        self._seed_t = None  # device-resident seed (CUDA-graph mode): kernels dereference it at run time
        self._draws = 0
        self._offset = 0
        self.param_epoch = 0
        self._shadows = {}
        self._static = {}
        self._static_grad = {}  # key -> fp32 view of the trainer's flat gradient buffer (direct accumulation)
        self._static_refresh = None  # callable that re-casts the owner's flat bf16 shadow from its fp32 master
        self._static_dirty = False   # fp32 parameters were written behind the owner's back (load_state_dict)
        self.attn_tensor_core = True  # bf16 mode: contractions of attention on the wgmma GEMM (else row kernels)
        self.attn_fused = True        # bf16 mode, Tk <= 320: single-launch fused forward (attention_flash.cu)
        self.attn_fused_bwd = True    # ... and the flash-style fused backward (attention_fused_bwd.cu)
        # set by incremental._attend: one-row, no-grad queries go to the split-KV decode kernel (attention_decode.cu)
        self.attn_decode_rows = False
        self.fold_residual_grad = os.environ.get("ST5_FOLD_RESGRAD", "1") != "0"  # see LinearFn.forward (passthrough)
        self.probs_grad_heads = 0     # > 0: gradients on returned probabilities exist for the first n heads only
        self.probs_read_heads = 0     # > 0: nobody READS returned probabilities beyond the first n heads (trainer, per step)
        # streaming forward for what the resident kernels cannot hold (Tk > 320, clipped relative positions); "all":
        # every bf16 shape goes through it (ST5_ATTN_FLASH=all)
        self.attn_flash = {"0": False, "all": "all"}.get(os.environ.get("ST5_ATTN_FLASH", "1"), True)
        self.ffn_gate = os.environ.get("ST5_FFN_GATE", "1") != "0"  # bf16 mode: fc1 stores the backward gate (FFNFn)
        self.wgrad_splitk = os.environ.get("ST5_WGRAD_SPLITK", "1") != "0"  # weight gradients: split-K + L2 reduce
        # out_proj / fc2 bias gradients come out of the consuming LayerNorm's backward pass (no column-sum launch)
        self.fold_bias_grad = os.environ.get("ST5_FOLD_BIAS_GRAD", "1") != "0"
        self.fp32_stream = os.environ.get("ST5_FP32_STREAM", "1") != "0"  # bf16 mode: fp32 residual stream between LayerNorms
        # trainer hooks: stage_callback(key, x) is called at the entry of every encoder / decoder layer (gradient-exchange
        # overlap point); layer_keep (device [n_enc + n_dec] 0/1 mask, CUDA-graph mode) / layer_keep_host (eager mode)
        # carry the trainer's LayerDrop draw -- when both are None the model draws for itself like the reference
        self.stage_callback = None
        self.layer_keep = None
        self.layer_keep_host = None
        # weight-gradient GEMMs on a second stream (trainer, single GPU, ST5_WGRAD_SIDE=1): see wgrad_mm / side_join
        self.wgrad_stream = None
        self._side_keep = []
        self.side_small = os.environ.get("ST5_SIDE_SMALL", "1") != "0"  # bias / table gradients ride on that stream too

    @property
    def seed(self):
        return self._seed_t.data_ptr() if self._seed_t is not None else self._seed

    def next_offset(self):
        self._offset += 1
        return (self._offset | self.SEED_PTR_FLAG) if self._seed_t is not None else self._offset

    def offset_block(self, base, i, width=64):
        """LayerDrop stacks: the dropout draws of layer i start at offset base + i * width, whether or not earlier
        layers ran. A captured update runs every layer and keeps or discards its output on the device, an eager one
        skips the dropped layers; with fixed blocks the layers both run draw the same masks (a layer draws < width)."""
        self._offset = base + i * width

    def manual_seed(self, seed):
        self._seed = int(seed)
        self._offset = 0
        self._draws = 0  # utterances synthesised since the last manual_seed (incremental.SynthesisGraph)
        if self._seed_t is not None:
            self._seed_t.fill_(self._seed)

    def enable_device_seed(self, device):
        """Keep the dropout seed in device memory so a captured graph draws new masks each replay."""
        if self._seed_t is None or self._seed_t.device != torch.device(device):
            self._seed_t = torch.full((1,), self._seed, dtype=torch.int64, device=device)

    def disable_device_seed(self):
        self._seed_t = None

    def advance_seed(self):
        """New dropout masks for the next step (device op; capturable)."""
        if self._seed_t is not None:
            self._seed_t += 1
        else:
            self._seed += 1
        self._offset = 0

    def side_join(self):
        """The main stream waits for every weight-gradient launch issued on the side stream; their operands may go."""
        if self.wgrad_stream is not None and self._side_keep:  # (only when something was issued there since the last
            torch.cuda.current_stream().wait_stream(self.wgrad_stream)  # join: a capture may not wait on foreign work)
        self._side_keep.clear()

    def stage(self, key, x):
        cb = self.stage_callback
        return x if cb is None else cb(key, x)

    def register_static(self, key, hi):
        """Shadow that is kept current by someone else (the trainer's flat bf16 buffer refreshed by the Adam kernel)."""
        self._static[key] = hi

    def register_static_refresh(self, fn):
        self._static_refresh = fn

    def register_static_grad(self, key, view):
        self._static_grad[key] = view

    def clear_static(self):
        self._static = {}
        self._static_grad = {}
        self._static_refresh = None
        self._static_dirty = False

    def invalidate_shadows(self):
        """Call after parameters change through the owner of the static shadows (optimizer step) or when there is none:
        cached per-parameter shadows are re-cast on next use."""
        self.param_epoch += 1

    def params_written_externally(self):
        """fp32 parameters were overwritten in place by someone who does not maintain the static bf16 shadows
        (load_state_dict after the trainer was built, manual edits): the next shadow() lookup re-casts the flat shadow
        from the fp32 master before handing out a view of it."""
        self.param_epoch += 1
        if self._static_refresh is not None:
            self._static_dirty = True

    def shadow(self, key, build):
        """bf16 (hi, lo) copy of a (possibly fused / re-laid-out) fp32 weight; `build()` returns the fp32 2-D tensor."""
        need_lo = self.dtype == torch.float32
        if self._static_dirty:
            self._static_dirty = False
            self._static_refresh()
        if not need_lo:
            st = self._static.get(key)
            if st is not None:
                return st, None
        ent = self._shadows.get(key)
        if ent is not None and ent[0] == self.param_epoch and (ent[2] is not None or not need_lo):
            return ent[1], ent[2]
        w = build()
        w = w.detach()
        if w.dim() != 2 or w.stride(1) != 1:
            w = w.reshape(w.shape[0], -1).contiguous()
        hi = torch.empty(w.shape, dtype=torch.bfloat16, device=w.device)
        lo = torch.empty_like(hi) if need_lo else None
        K.cast_bf16(w, hi, lo)
        self._shadows[key] = (self.param_epoch, hi, lo)
        return hi, lo


RT = Runtime()


def _split(x2d):
    """activation [rows, cols] (strided 2-D, unit inner stride) -> (hi, lo) bf16 operands for the GEMM."""
    if x2d.dtype == torch.bfloat16:
        return x2d, None
    rows, cols = x2d.shape
    ld = x2d.stride(0) if rows > 1 else _pad8(cols)  # keep the source row pitch: callers pass it as the GEMM ld
    hi = torch.empty((rows, ld), dtype=torch.bfloat16, device=x2d.device)[:, :cols]
    lo = torch.empty((rows, ld), dtype=torch.bfloat16, device=x2d.device)[:, :cols]
    K.cast_bf16(x2d, hi, lo)
    return hi, lo


def mm(a, b, out, *, M, N, Kd, a_mn=False, b_mn=False, a_ld=None, b_ld=None, c_ld=None, **epi):
    """out = epi(A . B^T) with A, B given as (hi, lo) pairs; lo is None in bf16 mode. Parity mode: 3 passes."""
    a_hi, a_lo = a
    b_hi, b_lo = b
    kw = dict(M=M, N=N, K=Kd, a_mn=a_mn, b_mn=b_mn, a_ld=a_ld, b_ld=b_ld, c_ld=c_ld)
    if a_lo is None and b_lo is None:
        return K.gemm(a_hi, b_hi, out, **kw, **epi)
    assert out.dtype == torch.float32, "split-precision GEMM accumulates in an fp32 output"
    acc0 = epi.pop("accumulate", False)
    alpha = epi.pop("alpha", 1.0)
    passes = [(a_hi, b_hi)]
    if b_lo is not None:
        passes.append((a_hi, b_lo))
    if a_lo is not None:
        passes.append((a_lo, b_hi))
    for i, (pa, pb) in enumerate(passes):
        last = i == len(passes) - 1
        K.gemm(pa, pb, out, **kw, alpha=alpha, accumulate=(acc0 or i > 0), **(epi if last else {}))
    return out


def _pad8(n):
    return (n + 7) // 8 * 8


def _off_critical_path(fn, *keep):
    """Run a launch whose result nothing reads before the optimizer (a gradient accumulated into the trainer's flat
    buffer) on the weight-gradient stream when the trainer opened one: the main chain does not wait for it, its operands
    are kept alive until RT.side_join()."""
    side = RT.wgrad_stream if RT.side_small else None
    if side is None:
        fn()
        return
    side.wait_stream(torch.cuda.current_stream())
    RT._side_keep.append(keep)
    with torch.cuda.stream(side):
        fn()


def _key_pad_u8(key_pad):
    """uint8 form of a key-padding mask. Every layer of a stack receives the SAME mask tensor: the converted copy rides
    on it as an attribute, so the cast runs once per forward pass instead of once per attention call (24 per update)."""
    if key_pad is None:
        return None
    if key_pad.dtype == torch.uint8 and key_pad.is_contiguous():
        return key_pad
    hit = getattr(key_pad, "_st5_u8", None)  # (version counter of the mask at conversion time, converted copy)
    if hit is not None and hit[0] == key_pad._version and hit[1].shape == key_pad.shape and hit[1].device == key_pad.device:
        return hit[1]
    u8 = key_pad.to(torch.uint8).contiguous()
    try:
        key_pad._st5_u8 = (key_pad._version, u8)
    except Exception:  # (tensor subclasses that refuse attributes)
        pass
    return u8


def _pe_bf16(pe_k):
    """bf16 copy of the relative-position table. A Parameter is cached per parameter epoch; a computed tensor (the
    pre-LN layers pass norm_k(table), transformer_layer.py:94-95) is cast every call -- its id() is not stable."""
    if isinstance(pe_k, torch.nn.Parameter):
        return RT.shadow(("pe", id(pe_k)), lambda: pe_k)[0]
    src = pe_k.detach()
    src = src if (src.dtype == torch.float32 and src.is_contiguous()) else src.float().contiguous()
    hi = torch.empty(src.shape, dtype=torch.bfloat16, device=src.device)
    K.cast_bf16(src, hi, None)
    return hi


def _resolve_act(act, dtype):
    """Throughput mode (bf16 activations) evaluates GELU in its tanh form on the MUFU unit (|error| <= 4.8e-4, below
    bf16 rounding of the result); parity mode (fp32) keeps the reference's exact erf form (fairseq/modules/gelu.py:24)."""
    return "gelu_tanh" if (act == "gelu" and dtype == torch.bfloat16) else act


def wgrad_mm(gy, gy_ld, xin, xin_ld, n_out, n_in, M, target=None):
    """dW[n_out, n_in] = gy^T . xin (both operands read MN-major, contraction over the M token rows).

    target != None: accumulate into that fp32 view of the flat gradient buffer and return None; else return a new dW.
    Small outputs (< half a wave of 128-wide tiles) with a long contraction are split along M into S partial products
    (the split rides on the GEMM's batch dimension: batch stride = chunk rows) that one column-sum launch reduces, so
    a 768x768 gradient uses ~8x more SMs than its 36 output tiles would."""
    dev = gy[0].device
    tiles = ((n_out + 127) // 128) * ((n_in + 127) // 128)
    S = 1
    splitk_l2 = (target is not None and gy[1] is None and xin[1] is None and RT.wgrad_splitk and n_out >= 256
                 and n_in >= 192 and target.is_contiguous() and target.data_ptr() % 16 == 0 and n_in % 4 == 0)
    if not splitk_l2 and gy[1] is None and xin[1] is None and tiles <= 72 and M >= 2048:
        for cand in (8, 6, 4, 3, 2):
            if cand * tiles <= 2 * 132 and M % cand == 0:  # at most two waves of 128 x 128 tiles
                S = cand
                break
    if S > 1:
        chunk = M // S
        parts = torch.empty((S, n_out, n_in), dtype=torch.float32, device=dev)
        K.gemm(gy[0], xin[0], parts, M=n_out, N=n_in, K=chunk, a_mn=True, a_ld=gy_ld, b_mn=True, b_ld=xin_ld,
               c_ld=n_in, nb1=S, nb2=1, a_bs=(chunk * gy_ld, 0), b_bs=(chunk * xin_ld, 0), c_bs=(n_out * n_in, 0))
        out = target if target is not None else torch.empty((n_out, n_in), dtype=torch.float32, device=dev)
        K.colsum(parts.view(S, n_out * n_in), out.view(-1), accumulate=target is not None)
        return None if target is not None else out
    if splitk_l2:
        # throughput mode, straight into the flat gradient buffer: the contraction split over the batch dimension so
        # that (128 x 128 tiles x splits) fills one wave of the 132 SMs, every partial product added to the gradient by
        # a TMA reduce at the L2 (nobody reads the gradient first, no partial buffers, no reduction launch). Splits
        # must divide M: a batch entry is a [chunk]-row window of the MN-major operands.
        S = 1
        for cand in (16, 12, 10, 8, 6, 5, 4, 3, 2):
            if cand * tiles <= 132 and M % cand == 0 and M // cand >= 512:
                S = cand
                break
        chunk = M // S
        side = RT.wgrad_stream
        if side is not None:
            # off the critical path: nothing downstream of this launch reads the gradient before the update, and the
            # TMA reduce-adds commute. A second stream lets it fill the SMs the main chain leaves idle at every kernel
            # boundary; the operands are kept alive until RT.side_join() (their memory must not be reused under it)
            side.wait_stream(torch.cuda.current_stream())
            RT._side_keep.append((gy[0], xin[0]))
            with torch.cuda.stream(side):
                K.gemm(gy[0], xin[0], target, M=n_out, N=n_in, K=chunk, a_mn=True, a_ld=gy_ld, b_mn=True, b_ld=xin_ld,
                       c_ld=n_in, nb1=S, nb2=1, a_bs=(chunk * gy_ld, 0), b_bs=(chunk * xin_ld, 0), c_bs=(0, 0), accumulate=2)
            return None
        K.gemm(gy[0], xin[0], target, M=n_out, N=n_in, K=chunk, a_mn=True, a_ld=gy_ld, b_mn=True, b_ld=xin_ld,
               c_ld=n_in, nb1=S, nb2=1, a_bs=(chunk * gy_ld, 0), b_bs=(chunk * xin_ld, 0), c_bs=(0, 0), accumulate=2)
        return None
    if target is not None:
        mm(gy, xin, target, M=n_out, N=n_in, Kd=M, a_mn=True, a_ld=gy_ld, b_mn=True, b_ld=xin_ld, c_ld=n_in,
           accumulate=True)
        return None
    dW = torch.empty((n_out, n_in), dtype=torch.float32, device=dev)
    mm(gy, xin, dW, M=n_out, N=n_in, Kd=M, a_mn=True, a_ld=gy_ld, b_mn=True, b_ld=xin_ld, c_ld=n_in)
    return dW


# =================================================================================================== Linear
class LinearFn(torch.autograd.Function):
    """y = dropout(act(x W^T + b (+ rowgroup bias))) (+ residual). W may be several parameters fused along N.

    Replaces nn.Linear call sites of the reference (multihead_attention.py:213-231,397; transformer_layer.py:127-132,
    385-391; speech_decoder_prenet.py:41-47,69-72; speech_decoder_postnet.py:31-32)."""

    @staticmethod
    def forward(ctx, x, residual, bias2, opts, *params):
        nw = opts["n_weights"]
        weights, biases = params[:nw], params[nw:]
        key = opts.get("key") or (("lin",) + tuple(id(w) for w in weights))
        w_sh = RT.shadow(key, (lambda: weights[0]) if nw == 1 else (lambda: torch.cat([w.detach() for w in weights], 0)))
        N, Kd = w_sh[0].shape
        x2 = x.reshape(-1, x.shape[-1])
        M = x2.shape[0]
        assert x2.shape[1] == Kd and x2.stride(1) == 1
        bias = None
        if len(biases) > 0:
            bias = RT._static.get(("bias",) + tuple(id(b) for b in biases))  # contiguous view of the flat buffer
            if bias is None:
                bias = biases[0].detach() if len(biases) == 1 else torch.cat([b.detach() for b in biases], 0)
                bias = bias.float().contiguous()
        ldc = _pad8(N)
        out_dtype = opts.get("out_dtype", x.dtype)
        out = torch.empty((M, ldc), dtype=out_dtype, device=x.device)
        act, drop_p = _resolve_act(opts.get("act"), out.dtype), opts.get("drop_p", 0.0)
        pre = torch.empty_like(out) if act is not None else None
        off = RT.next_offset() if drop_p > 0 else 0
        xa = _split(x2)
        res2 = residual.reshape(M, -1) if residual is not None else None
        if res2 is not None:
            assert res2.shape[1] == N and ldc == N and res2.is_contiguous()
        mm(xa, w_sh, out, M=M, N=N, Kd=Kd, a_ld=x2.stride(0), b_ld=Kd, c_ld=ldc, bias=bias,
           bias2=bias2.detach().float().contiguous() if bias2 is not None else None,
           bias2_rows=opts.get("bias2_rows", 0), residual=res2, c_pre=pre, act=act, drop_p=drop_p, seed=RT.seed,
           offset=off)
        ctx.save_for_backward(x2, pre)
        ctx.bias_holder = opts.get("bias_holder")
        ctx.meta = (weights, biases, w_sh, xa if x2.dtype == torch.float32 else None, act, drop_p, off, N, Kd, M, ldc,
                    x.shape, residual is not None, bias2 is not None, opts.get("bias2_rows", 0), RT.seed,
                    opts.get("need_dx", True))
        y = out if ldc == N else out[:, :N]
        y = y.reshape(*x.shape[:-1], N)
        if opts.get("passthrough"):
            # second output = the input itself (an alias). The caller uses IT, not x, for the block's residual add: the
            # gradient of the residual branch then arrives HERE, next to dy, and is added in the epilogue of the dx GEMM
            # instead of by a separate elementwise kernel in autograd's accumulation (one launch + 3 tensor passes per block)
            ctx.set_materialize_grads(False)
            return y, x.view_as(x)
        return y

    @staticmethod
    def backward(ctx, dy, d_pt=None):
        x2, pre = ctx.saved_tensors
        (weights, biases, w_sh, xa, act, drop_p, off, N, Kd, M, ldc, xshape, has_res, has_b2, b2rows, seed,
         need_dx) = ctx.meta
        if dy is None:  # (passthrough form: only the residual branch carried a gradient)
            dy = torch.zeros((M, N), dtype=x2.dtype, device=x2.device)
        dev = dy.device
        if dy.dtype != x2.dtype:  # fp32 head outputs of a bf16 network: gradients re-enter the bf16 stream here
            dy = dy.to(x2.dtype)
        dy2 = dy.reshape(M, N)
        if not (dy2.stride(1) == 1 and dy2.stride(0) % 8 == 0 and dy2.data_ptr() % 16 == 0):
            buf = torch.zeros((M, ldc), dtype=dy.dtype, device=dev)
            buf[:, :N] = dy2
            dy2 = buf[:, :N]
        d_res = dy if has_res else None
        if act is not None or drop_p > 0:
            dpre_full = torch.empty((M, dy2.stride(0)), dtype=dy.dtype, device=dev)
            if act is not None:
                # elementwise over the padded row pitch: indices must match the forward's logical (m * N + n) index
                if dy2.stride(0) == N and ldc == N:
                    K.act_bwd(dy2, pre, dpre_full, act, drop_p, seed, off)
                else:
                    dyc = dy2.contiguous()
                    prec = pre[:, :N].contiguous()
                    tmp = torch.empty_like(dyc)
                    K.act_bwd(dyc, prec, tmp, act, drop_p, seed, off)
                    dpre_full = torch.zeros((M, ldc), dtype=dy.dtype, device=dev)
                    dpre_full[:, :N] = tmp
            else:
                dyc = dy2.contiguous()
                tmp = torch.empty_like(dyc)
                K.dropout(dyc, tmp, drop_p, seed, off)
                dpre_full = torch.zeros((M, ldc), dtype=dy.dtype, device=dev)
                dpre_full[:, :N] = tmp
            dpre = dpre_full[:, :N]
        else:
            dpre = dy2
        ga = _split(dpre)
        dpre_ld = dpre.stride(0)
        dx = None
        if need_dx and ctx.needs_input_grad[0]:
            dx = torch.empty((M, Kd), dtype=dy.dtype, device=dev)
            r_pt = None
            if d_pt is not None:
                r_pt = d_pt.reshape(M, Kd)
                r_pt = r_pt if (r_pt.is_contiguous() and r_pt.dtype == dx.dtype) else r_pt.to(dx.dtype).contiguous()
            # dx[m,k] = sum_n dpre[m,n] W[n,k] (+ the residual branch's gradient): B rows = k, stored [n][k] -> MN-major
            mm(ga, w_sh, dx, M=M, N=Kd, Kd=N, a_ld=dpre_ld, b_mn=True, b_ld=Kd, c_ld=Kd, residual=r_pt)
            dx = dx.reshape(xshape)
        elif d_pt is not None:
            dx = d_pt
        # dW[n,k] = sum_m dpre[m,n] x[m,k]: both operands MN-major. When the trainer owns a flat gradient buffer the
        # GEMM accumulates straight into it (fused group = one contiguous [N,K] region) and autograd gets None.
        xop = xa if xa is not None else (x2, None)
        gW = RT._static_grad.get(("lin",) + tuple(id(w) for w in weights))
        dW = wgrad_mm(ga, dpre_ld, xop, x2.stride(0), N, Kd, M, target=gW)
        if dW is None:
            grads_w = [None] * len(weights)
        else:
            grads_w, r0 = [], 0
            for w in weights:
                grads_w.append(dW[r0:r0 + w.shape[0]].reshape(w.shape))
                r0 += w.shape[0]
        grads_b = []
        d_b2 = None
        holder = ctx.bias_holder
        if len(biases) > 0 or has_b2:
            if len(biases) > 0 and holder is not None and holder["taken"]:
                # the LayerNorm that consumed y already summed the columns of its dx (= dpre) in its own backward pass
                db = holder["value"]
                if db is None:
                    grads_b = [None] * len(biases)
                else:
                    r0 = 0
                    for b in biases:
                        grads_b.append(db[r0:r0 + b.shape[0]])
                        r0 += b.shape[0]
            elif len(biases) > 0:
                gB = RT._static_grad.get(("bias",) + tuple(id(b) for b in biases))
                if gB is not None:
                    _off_critical_path(lambda: K.colsum(dpre, gB, ld=dpre_ld, accumulate=True), dpre, dy)
                    grads_b = [None] * len(biases)
                else:
                    db = torch.empty(N, dtype=torch.float32, device=dev)
                    K.colsum(dpre, db, ld=dpre_ld)
                    r0 = 0
                    for b in biases:
                        grads_b.append(db[r0:r0 + b.shape[0]])
                        r0 += b.shape[0]
            if has_b2:
                d_b2 = torch.empty(((M + b2rows - 1) // b2rows, N), dtype=torch.float32, device=dev)
                K.colsum(dpre, d_b2, group_rows=b2rows, ld=dpre_ld)
        return (dx, d_res, d_b2, None, *grads_w, *grads_b)


def _alias_with_stream(x_pt, x):
    f32 = getattr(x, "_st5_f32", None)  # the fp32 copy of the residual stream rides along (residual_layer_norm)
    if f32 is not None:
        x_pt._st5_f32 = f32
    return x_pt


def _bias_holder(biases):
    """Hand-over of a bias gradient to the LayerNorm that consumes the projection's output (residual_layer_norm picks it
    up from the tensor): its backward pass sums the columns of its dx anyway-resident rows, so the projection's own
    column-sum launch is skipped. `taken` stays False when nobody picked it up (the projection then sums itself)."""
    return dict(taken=False, value=None, key=("bias",) + tuple(id(b) for b in biases), n=sum(b.shape[0] for b in biases))


def linear(x, weights, biases=(), *, act=None, drop_p=0.0, residual=None, bias2=None, bias2_rows=0, out_dtype=None,
           need_dx=True, key=None, passthrough=False, bias_grad_by_consumer=False):
    if isinstance(weights, torch.Tensor):
        weights = (weights,)
    if isinstance(biases, torch.Tensor):
        biases = (biases,)
    biases = tuple(b for b in biases if b is not None)
    opts = dict(n_weights=len(weights), act=act, drop_p=drop_p, bias2_rows=bias2_rows, need_dx=need_dx, key=key,
                passthrough=bool(passthrough))
    if out_dtype is not None:
        opts["out_dtype"] = out_dtype
    holder = None
    if (bias_grad_by_consumer and len(biases) > 0 and act is None and drop_p == 0.0 and residual is None
            and torch.is_grad_enabled() and RT.fold_bias_grad):
        holder = opts["bias_holder"] = _bias_holder(biases)
    if passthrough:  # (y, alias of x for the caller's residual add: see LinearFn.forward)
        y, x_pt = LinearFn.apply(x, residual, bias2, opts, *weights, *biases)
        return y, _alias_with_stream(x_pt, x)
    y = LinearFn.apply(x, residual, bias2, opts, *weights, *biases)
    if holder is not None:
        y._st5_bias_holder = holder
    return y


class FFNFn(torch.autograd.Function):
    """o = dropout_o(fc2(dropout_a(act(fc1(x))))) (+ residual): the position-wise FFN of transformer_layer.py:127-132 /
    :385-391 as two GEMMs whose epilogues carry bias, GELU (+ pre-activation store) and dropout; in backward the
    activation/dropout derivative is fused into the epilogue of the dH = dO.W2 GEMM (no elementwise pass over
    [rows, ffn])."""

    @staticmethod
    def forward(ctx, x, residual, w1, b1, w2, b2, act, drop_a, drop_o, passthrough=False, bias_holder=None):
        ctx.bias_holder = bias_holder
        x2 = x.reshape(-1, x.shape[-1])
        M, D = x2.shape
        F_ = w1.shape[0]
        act = _resolve_act(act, x.dtype)
        w1s, w2s = RT.shadow(("lin", id(w1)), lambda: w1), RT.shadow(("lin", id(w2)), lambda: w2)
        bb1 = RT._static.get(("bias", id(b1)), None)
        bb1 = bb1 if bb1 is not None else b1.detach().float().contiguous()
        bb2 = RT._static.get(("bias", id(b2)), None)
        bb2 = bb2 if bb2 is not None else b2.detach().float().contiguous()
        h = torch.empty((M, F_), dtype=x.dtype, device=x.device)
        pre = torch.empty_like(h)
        off_a = RT.next_offset() if drop_a > 0 else 0
        xa = _split(x2)
        # throughput mode: the fc1 epilogue stores the backward GATE keep * scale * gelu'(pre) in place of the
        # pre-activation (tanh(u) is shared with the forward value), so the dH GEMM's epilogue is a single multiply
        gate = act == "gelu_tanh" and x.dtype == torch.bfloat16 and F_ % 8 == 0 and RT.ffn_gate
        mm(xa, w1s, h, M=M, N=F_, Kd=D, a_ld=x2.stride(0), b_ld=D, c_ld=F_, bias=bb1, c_pre=pre,
           act="gelu_tanh_gate" if gate else act, drop_p=drop_a, seed=RT.seed, offset=off_a)
        if gate:
            act = "gate"
        o = torch.empty((M, D), dtype=x.dtype, device=x.device)
        off_o = RT.next_offset() if drop_o > 0 else 0
        res2 = residual.reshape(M, D).contiguous() if residual is not None else None
        ha = _split(h)
        mm(ha, w2s, o, M=M, N=D, Kd=F_, a_ld=F_, b_ld=F_, c_ld=D, bias=bb2, residual=res2, drop_p=drop_o, seed=RT.seed,
           offset=off_o)
        ctx.save_for_backward(x2, h, pre)
        ctx.meta = (w1, b1, w2, b2, w1s, w2s, act, drop_a, off_a, drop_o, off_o, RT.seed, x.shape, residual is not None,
                    xa if x2.dtype == torch.float32 else None, ha if x2.dtype == torch.float32 else None)
        if passthrough:  # (o, alias of x): the residual branch's gradient comes back into this backward (LinearFn.forward)
            ctx.set_materialize_grads(False)
            return o.reshape(x.shape), x.view_as(x)
        return o.reshape(x.shape)

    @staticmethod
    def backward(ctx, do, d_pt=None):
        x2, h, pre = ctx.saved_tensors
        (w1, b1, w2, b2, w1s, w2s, act, drop_a, off_a, drop_o, off_o, seed, xshape, has_res, xa, ha) = ctx.meta
        M, D = x2.shape
        F_ = h.shape[1]
        if do is None:
            do = torch.zeros(xshape, dtype=x2.dtype, device=x2.device)
        dev = do.device
        do2 = do.reshape(M, D).contiguous()
        d_res = do if has_res else None
        if drop_o > 0:
            tmp = torch.empty_like(do2)
            K.dropout(do2, tmp, drop_o, seed, off_o)
            do2 = tmp
        ga = _split(do2)
        # dH_pre = (dO W2) * dropmask_a * act'(pre)  -- fused into the GEMM epilogue
        dhp = torch.empty((M, F_), dtype=do.dtype, device=dev)
        mm(ga, w2s, dhp, M=M, N=F_, Kd=D, a_ld=D, b_mn=True, b_ld=F_, c_ld=F_, drop_p=0.0 if act == "gate" else drop_a,
           seed=seed, offset=off_a, actgrad_pre=pre, actgrad_act=act)
        gh = _split(dhp)

        def wgrad(gy, gy_ld, xin, xin_ld, w, n_out, n_in):
            return wgrad_mm(gy, gy_ld, xin, xin_ld, n_out, n_in, M, target=RT._static_grad.get(("lin", id(w))))

        def bgrad(gy2d, b):
            gB = RT._static_grad.get(("bias", id(b)))
            if gB is not None:
                _off_critical_path(lambda: K.colsum(gy2d, gB, accumulate=True), gy2d)
                return None
            db = torch.empty(b.shape[0], dtype=torch.float32, device=dev)
            K.colsum(gy2d, db)
            return db

        dW2 = wgrad(ga, D, ha if ha is not None else (h, None), F_, w2, D, F_)
        holder = ctx.bias_holder
        if holder is not None and holder["taken"]:  # summed by the consuming LayerNorm's backward (see _bias_holder)
            db2 = holder["value"]
        else:
            db2 = bgrad(do2, b2)
        dW1 = wgrad(gh, F_, xa if xa is not None else (x2, None), x2.stride(0), w1, F_, D)
        db1 = bgrad(dhp, b1)
        dx = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty((M, D), dtype=do.dtype, device=dev)
            r_pt = None
            if d_pt is not None:
                r_pt = d_pt.reshape(M, D)
                r_pt = r_pt if (r_pt.is_contiguous() and r_pt.dtype == dx.dtype) else r_pt.to(dx.dtype).contiguous()
            mm(gh, w1s, dx, M=M, N=D, Kd=F_, a_ld=F_, b_mn=True, b_ld=D, c_ld=D, residual=r_pt)
            dx = dx.reshape(xshape)
        elif d_pt is not None:
            dx = d_pt
        return dx, d_res, dW1, db1, dW2, db2, None, None, None, None, None


def ffn(x, fc1, fc2, act, drop_a=0.0, drop_o=0.0, residual=None, passthrough=False, bias_grad_by_consumer=False):
    holder = None
    if (bias_grad_by_consumer and drop_o == 0.0 and residual is None and fc2.bias is not None and torch.is_grad_enabled()
            and RT.fold_bias_grad):
        holder = _bias_holder((fc2.bias,))
    if passthrough:
        o, x_pt = FFNFn.apply(x, residual, fc1.weight, fc1.bias, fc2.weight, fc2.bias, act, drop_a, drop_o, True, holder)
        if holder is not None:
            o._st5_bias_holder = holder
        return o, _alias_with_stream(x_pt, x)
    o = FFNFn.apply(x, residual, fc1.weight, fc1.bias, fc2.weight, fc2.bias, act, drop_a, drop_o, False, holder)
    if holder is not None:
        o._st5_bias_holder = holder
    return o


# =================================================================================================== LayerNorm
class ResidualLayerNormFn(torch.autograd.Function):
    """y = LayerNorm(residual + dropout(x)) -- the post-LN tail of every reference block
    (transformer_layer.py:112-132, 343-391) and the encoder input LayerNorm (encoder.py:226-227)."""

    @staticmethod
    def forward(ctx, x, residual, gamma, beta, eps, drop_p, res_f32=None, y_f32=None, bias_holder=None):
        ctx.bias_holder = bias_holder
        x = x.contiguous()
        Cc = x.shape[-1]
        rows = x.numel() // Cc
        y = torch.empty_like(x)
        s = torch.empty_like(x)
        mean = torch.empty(rows, dtype=torch.float32, device=x.device)
        rstd = torch.empty_like(mean)
        off = RT.next_offset() if drop_p > 0 else 0
        res = residual.contiguous() if residual is not None else None
        K.ln_fwd(x, res, gamma.detach(), beta.detach(), y, s, mean, rstd, eps, drop_p, RT.seed, off,
                 residual_f32=res_f32, y_f32=y_f32)
        ctx.save_for_backward(s, mean, rstd, gamma)
        ctx.meta = (drop_p, off, RT.seed, residual is not None, id(gamma), id(beta))
        return y

    @staticmethod
    def backward(ctx, dy):
        s, mean, rstd, gamma = ctx.saved_tensors
        drop_p, off, seed, has_res, gid, bid = ctx.meta
        dy = dy.contiguous()
        ds = torch.empty_like(dy)
        dx = torch.empty_like(dy) if drop_p > 0 else None
        # the parameter-gradient kernel adds its partial sums atomically: aim it at the flat gradient buffer when the
        # trainer registered one (zeroed at the start of the update), else at fresh zero vectors handed to autograd
        gG, gB = RT._static_grad.get(("bias", gid)), RT._static_grad.get(("bias", bid))
        direct = gG is not None and gB is not None
        dgamma = gG if direct else torch.zeros_like(gamma, dtype=torch.float32)
        dbeta = gB if direct else torch.zeros_like(gamma, dtype=torch.float32)
        holder, dxsum = ctx.bias_holder, None
        if holder is not None:  # the producing projection's bias gradient = column sums of dx (see ops._bias_holder)
            dxsum = RT._static_grad.get(holder["key"])
            if dxsum is None:
                dxsum = holder["value"] = torch.zeros(holder["n"], dtype=torch.float32, device=dy.device)
            holder["taken"] = True
        K.ln_bwd(dy, s, mean, rstd, gamma.detach(), ds, dx, dgamma, dbeta, drop_p, seed, off, dxsum=dxsum)
        if direct:
            dgamma = dbeta = None
        return (dx if dx is not None else ds), (ds if has_res else None), dgamma, dbeta, None, None, None, None, None


def _layer_norm_wide(x, residual, ln):
    """LayerNorm(x + residual) over rows of 1024 < C <= 2048 channels on st5_ln_fwd_wide: evaluation only."""
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in (x, residual, ln.weight, ln.bias)):
        raise NotImplementedError(f"LayerNorm over {x.shape[-1]} channels has no backward (training takes C <= 1024)")
    x = x.contiguous()
    y = torch.empty_like(x)
    K.ln_fwd_wide(x, residual.contiguous() if residual is not None else None, ln.weight.detach(), ln.bias.detach(), y,
                  eps=ln.eps)
    return y


def residual_layer_norm(x, residual, ln, drop_p=0.0, stream=False):
    """stream=True (post-LN blocks, throughput mode): keep an fp32 copy of the output next to the bf16 activations and
    feed it to the next block's residual add, so that the residual stream is never rounded to bf16 between layers. The
    copy rides along as a plain attribute of the returned tensor (no autograd node: gradients flow through the bf16
    tensor exactly as before)."""
    if x.shape[-1] > 1024:  # (st5_ln_fwd takes C <= 1024; wider rows have a forward-only kernel)
        assert drop_p == 0.0
        return _layer_norm_wide(x, residual, ln)
    res_f32 = getattr(residual, "_st5_f32", None) if residual is not None else None
    y_f32 = None
    if stream and RT.fp32_stream and x.dtype == torch.bfloat16 and x.is_cuda:
        y_f32 = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    if res_f32 is not None and (res_f32.shape != x.shape or not res_f32.is_contiguous()):
        res_f32 = None
    holder = getattr(x, "_st5_bias_holder", None)
    if holder is not None and (holder["n"] != x.shape[-1] or not torch.is_grad_enabled()):
        holder = None
    y = ResidualLayerNormFn.apply(x, residual, ln.weight, ln.bias, ln.eps, drop_p, res_f32, y_f32, holder)
    if y_f32 is not None:
        y._st5_f32 = y_f32
    return y


# =================================================================================================== pos. encoding
class PosEncFn(torch.autograd.Function):
    """dropout((E[tokens] | x) + alpha * pe): text_encoder_prenet.py:36-45, speech_decoder_prenet.py:52-67."""

    @staticmethod
    def forward(ctx, tokens, emb, x, pe, alpha, padding_idx, drop_p):
        if tokens is not None:
            B, T = tokens.shape
            Cc = emb.shape[1]
            y = torch.empty((B, T, Cc), dtype=RT.dtype, device=emb.device)
        else:
            x = x.contiguous()
            B, T, Cc = x.shape
            y = torch.empty_like(x)
        off = RT.next_offset() if drop_p > 0 else 0
        K.posenc_fwd(tokens, emb.detach() if emb is not None else None, x, pe, alpha.detach(), y, drop_p, RT.seed, off)
        ctx.save_for_backward(tokens, pe)
        ctx.meta = (emb.shape if emb is not None else None, padding_idx, drop_p, off, RT.seed, x is not None)
        return y

    @staticmethod
    def backward(ctx, dy):
        tokens, pe = ctx.saved_tensors
        emb_shape, padding_idx, drop_p, off, seed, has_x = ctx.meta
        dy = dy.contiguous()
        dx = torch.empty_like(dy) if has_x else None
        demb = torch.zeros(emb_shape, dtype=torch.float32, device=dy.device) if emb_shape is not None else None
        dalpha = torch.zeros((), dtype=torch.float32, device=dy.device)
        K.posenc_bwd(dy, tokens, padding_idx if padding_idx is not None else -1, pe, dx, demb, dalpha, drop_p, seed, off)
        return None, demb, dx, None, dalpha, None, None


def scaled_posenc(pe, alpha, drop_p, tokens=None, emb=None, padding_idx=None, x=None):
    return PosEncFn.apply(tokens, emb, x, pe, alpha, padding_idx, drop_p)


# =================================================================================================== attention
class AttentionFn(torch.autograd.Function):
    """softmax(scale * q (k + pe)^T + masks) v on fused projection buffers.

    q_buf: [B, Tq, nq*d] with q in column block `q_col`; kv_buf: [B, Tk, nk*d] with k / v in blocks k_col / v_col
    (kv_buf is q_buf for self-attention). Returns (out [B,Tq,d], probs [B,H,Tq,p_ld] fp32 or activation dtype)."""

    @staticmethod
    def forward(ctx, q_buf, kv_buf, pe_k, key_pad, cfg):
        ctx.set_materialize_grads(False)
        same = kv_buf is None
        kvb = q_buf if same else kv_buf
        B, Tq = q_buf.shape[0], q_buf.shape[1]
        Tk = kvb.shape[1]
        H, d = cfg["H"], cfg["d"]
        assert d == H * 64
        dev = q_buf.device
        out = torch.empty((B, Tq, d), dtype=q_buf.dtype, device=dev)
        p_ld = _pad8(Tk)
        probs_dtype = torch.float32 if cfg.get("return_probs") else q_buf.dtype
        probs = torch.empty((B, H, Tq, p_ld), dtype=probs_dtype, device=dev)
        drop_p = cfg.get("drop_p", 0.0)
        off = RT.next_offset() if drop_p > 0 else 0
        kp = _key_pad_u8(key_pad)
        esz = q_buf.element_size()
        common = dict(
            B=B, H=H, Tq=Tq, Tk=Tk, dtype=K.dtype_id(q_buf), causal=int(cfg.get("causal", False)),
            maxpos=cfg.get("maxpos", 0), probs_dtype=K.dtype_id(probs),
            q=q_buf.data_ptr() + cfg["q_col"] * d * esz, q_ld=q_buf.stride(1), q_bs=q_buf.stride(0),
            k=kvb.data_ptr() + cfg["k_col"] * d * esz, k_ld=kvb.stride(1), k_bs=kvb.stride(0),
            v=kvb.data_ptr() + cfg["v_col"] * d * esz, v_ld=kvb.stride(1), v_bs=kvb.stride(0),
            key_pad=kp, pe_k=pe_k.detach() if pe_k is not None else None,
            out=out, o_ld=d, o_bs=Tq * d, probs=probs, p_ld=p_ld,
            scale=cfg["scale"], drop_p=drop_p, seed=RT.seed, offset=off)
        K.attn_fwd(K.attn_args(**common))
        ctx.save_for_backward(q_buf, kv_buf, pe_k, kp, probs)
        ctx.meta = (cfg, off, RT.seed, p_ld, same)
        return out, probs[..., :Tk] if p_ld != Tk else probs

    @staticmethod
    def backward(ctx, dout, dprobs):
        q_buf, kv_buf, pe_k, kp, probs = ctx.saved_tensors
        cfg, off, seed, p_ld, same = ctx.meta
        kvb = q_buf if same else kv_buf
        B, Tq = q_buf.shape[0], q_buf.shape[1]
        Tk = kvb.shape[1]
        H, d = cfg["H"], cfg["d"]
        dev = q_buf.device
        if dout is None:
            dout = torch.zeros((B, Tq, d), dtype=q_buf.dtype, device=dev)
        dout = dout.contiguous()
        dq_buf = torch.zeros_like(q_buf) if q_buf.shape[2] != (3 * d if same else d) else torch.empty_like(q_buf)
        dkv_buf = dq_buf if same else torch.empty_like(kv_buf)
        ds = torch.empty((B, H, Tq, p_ld), dtype=torch.float32, device=dev)
        dpe = torch.zeros_like(pe_k, dtype=torch.float32) if pe_k is not None else None
        dpx = None
        if dprobs is not None:
            dpx = dprobs
            if dpx.dtype != torch.float32 or dpx.shape[-1] != p_ld or not dpx.is_contiguous():
                buf = torch.zeros((B, H, Tq, p_ld), dtype=torch.float32, device=dev)
                buf[..., :Tk] = dprobs
                dpx = buf
        esz = q_buf.element_size()
        a = K.attn_args(
            B=B, H=H, Tq=Tq, Tk=Tk, dtype=K.dtype_id(q_buf), causal=int(cfg.get("causal", False)),
            maxpos=cfg.get("maxpos", 0), probs_dtype=K.dtype_id(probs),
            q=q_buf.data_ptr() + cfg["q_col"] * d * esz, q_ld=q_buf.stride(1), q_bs=q_buf.stride(0),
            k=kvb.data_ptr() + cfg["k_col"] * d * esz, k_ld=kvb.stride(1), k_bs=kvb.stride(0),
            v=kvb.data_ptr() + cfg["v_col"] * d * esz, v_ld=kvb.stride(1), v_bs=kvb.stride(0),
            key_pad=kp, pe_k=pe_k.detach() if pe_k is not None else None,
            out=None, o_ld=d, o_bs=Tq * d, probs=probs, p_ld=p_ld, scale=cfg["scale"],
            drop_p=cfg.get("drop_p", 0.0), seed=seed, offset=off,
            dout=dout, dprobs_ext=dpx, ds=ds,
            dq=dq_buf.data_ptr() + cfg["q_col"] * d * esz, dk=dkv_buf.data_ptr() + cfg["k_col"] * d * esz,
            dv=dkv_buf.data_ptr() + cfg["v_col"] * d * esz, dpe_k=dpe)
        K.attn_bwd(a)
        return dq_buf, (None if same else dkv_buf), dpe, None, None


class AttentionTCFn(torch.autograd.Function):
    """bf16 tensor-core attention: every contraction (QK^T, Q.PE^T, PV and the five backward products) is a batched
    launch of the wgmma GEMM over (head, utterance) reading q/k/v in place from the fused projection buffers; the
    softmax / dS / relative-position scatter steps are the row kernels of csrc/attention_tc.cu. Same interface and
    dropout-mask convention as AttentionFn (the exact fp32 row-kernel path used for parity mode)."""

    @staticmethod
    def _fused_backward(q_buf, kv_buf, probs, cfg, off, seed, p_ld, same, fused, dout, dprobs):
        """One launch (+ the row-constant pre-pass): flash-style backward on wgmma (attention_fused_bwd.cu). `fused` =
        (out, psave, inv_l, key_pad): psave / inv_l are the exponentials (dropout decision in the sign bit) and the row
        normalisers the forward saved; `probs` the fp32 probabilities it returned to the caller (only with dprobs)."""
        out, psave, inv_l, o32, kp = fused
        kvb = q_buf if same else kv_buf
        B, Tq, Tk = q_buf.shape[0], q_buf.shape[1], kvb.shape[1]
        H, d = cfg["H"], cfg["d"]
        dev = q_buf.device
        if dout is None:
            dout = torch.zeros((B, Tq, d), dtype=torch.bfloat16, device=dev)
        dout = dout.contiguous()
        qv, kk, vv = AttentionTCFn._views(q_buf, kvb, cfg)
        full = q_buf.shape[2] == (3 * d if same else d)
        dq_buf = torch.empty_like(q_buf) if full else torch.zeros_like(q_buf)
        dkv_buf = dq_buf if same else torch.empty_like(kv_buf)
        dqv, dkk, dvv = AttentionTCFn._views(dq_buf, dkv_buf, cfg)
        dpx = None
        if dprobs is not None:
            assert probs is not None and probs.dtype == torch.float32, "external dP needs the returned fp32 probabilities"
            dpx = dprobs
            if dpx.dtype != torch.float32 or dpx.shape[-1] != p_ld or not dpx.is_contiguous():
                buf = torch.zeros((B, H, Tq, p_ld), dtype=torch.float32, device=dev)
                buf[..., :Tk] = dprobs
                dpx = buf
        delta = torch.empty((B, H, Tq), dtype=torch.float32, device=dev)
        dq_acc = torch.empty((B, Tq, d), dtype=torch.float32, device=dev)
        a = K.attn_args(B=B, H=H, Tq=Tq, Tk=Tk, dtype=K.dtype_id(q_buf), causal=int(cfg.get("causal", False)), maxpos=0,
                        probs_dtype=K.dtype_id(probs) if probs is not None else 0, q=qv, q_ld=q_buf.stride(1),
                        q_bs=q_buf.stride(0), k=kk, k_ld=kvb.stride(1),
                        k_bs=kvb.stride(0), v=vv, v_ld=kvb.stride(1), v_bs=kvb.stride(0), key_pad=kp, pe_k=None,
                        out=out, o_ld=d, o_bs=Tq * d, probs=probs if dpx is not None else None, p_ld=p_ld,
                        scale=cfg["scale"], drop_p=cfg.get("drop_p", 0.0), seed=seed, offset=off, dout=dout,
                        dprobs_ext=dpx, ds=None, dq=dqv, dk=dkk, dv=dvv, dpe_k=None)
        K.attn_fused_bwd(a, psave, inv_l, o32, delta, dq_acc, ext_heads=cfg.get("probs_grad_heads", 0) if dpx is not None else 0)
        return dq_buf, (None if same else dkv_buf), None, None, None

    @staticmethod
    def _fused_backward_rpe(q_buf, pe_k, pe_hi, cfg, off, seed, p_ld, fused, dout, dprobs):
        """Relative-position self-attention: the fused kernel (saved exponentials read back, dS written) + the two
        table contractions."""
        assert dprobs is None, "external dP is not supported together with relative positions"
        out, psave, inv_l, o32, kp = fused
        B, Tq, _ = q_buf.shape
        Tk = Tq
        H, d, scale, maxpos = cfg["H"], cfg["d"], cfg["scale"], cfg["maxpos"]
        dev = q_buf.device
        if dout is None:
            dout = torch.zeros((B, Tq, d), dtype=torch.bfloat16, device=dev)
        dout = dout.contiguous()
        qv, kk, vv = AttentionTCFn._views(q_buf, q_buf, cfg)
        q_ld, q_bs = q_buf.stride(1), q_buf.stride(0)
        full = q_buf.shape[2] == 3 * d
        dq_buf = torch.empty_like(q_buf) if full else torch.zeros_like(q_buf)
        dqv, dkk, dvv = AttentionTCFn._views(dq_buf, dq_buf, cfg)
        delta = torch.empty((B, H, Tq), dtype=torch.float32, device=dev)
        dq_acc = torch.empty((B, Tq, d), dtype=torch.float32, device=dev)
        dS = torch.empty((B, H, Tq, p_ld), dtype=torch.bfloat16, device=dev)
        a = K.attn_args(B=B, H=H, Tq=Tq, Tk=Tk, dtype=K.dtype_id(q_buf), causal=0, maxpos=maxpos,
                        probs_dtype=0, q=qv, q_ld=q_ld, q_bs=q_bs, k=kk, k_ld=q_ld, k_bs=q_bs, v=vv,
                        v_ld=q_ld, v_bs=q_bs, key_pad=kp, pe_k=pe_hi, out=out, o_ld=d, o_bs=Tq * d, probs=None, p_ld=p_ld,
                        scale=scale, drop_p=cfg.get("drop_p", 0.0), seed=seed, offset=off, dout=dout, dprobs_ext=None,
                        ds=dS, dq=dqv, dk=dkk, dv=dvv, dpe_k=None)
        K.attn_fused_bwd(a, psave, inv_l, o32, delta, dq_acc)
        R = pe_k.shape[0]
        rows = B * Tq
        if q_bs == Tq * q_ld and RT.wgrad_splitk:
            # head-major dQP: one head's rows (b, i) are equidistant in dQP and in the fused q|k|v buffer, so the two
            # table contractions are 12 long GEMMs (M or K = B*T) instead of B x H short ones whose second 128-row tile
            # is three quarters empty at T = 160
            dQP = torch.empty((H, B, Tq, R), dtype=torch.bfloat16, device=dev)
            K.attn_dqp_scatter(dS, dQP, B, H, Tq, Tk, p_ld, maxpos, h_major=True)
            # dQ += scale dQP PE
            K.gemm(dQP, pe_hi, dqv, M=rows, N=64, K=R, a_ld=R, b_mn=True, b_ld=64, c_ld=q_ld, nb1=H, nb2=1,
                   a_bs=(rows * R, 0), b_bs=(0, 0), c_bs=(64, 0), alpha=scale, residual=dqv)
            # dPE[r,c] = scale sum_{h} sum_{b,i} dQP[h,b,i,r] q[b,i,h,c]: heads and contraction splits all add into one
            # [R, 64] output at the L2
            S = next((c for c in (8, 6, 5, 4, 3, 2) if rows % c == 0 and rows // c >= 512), 1)
            chunk = rows // S
            # (straight into the trainer's flat gradient buffer when the table is a registered parameter: no zero fill,
            # no AccumulateGrad add per layer -- the 12 encoder layers share ONE table)
            target = RT._static_grad.get(("lin", id(pe_k))) if isinstance(pe_k, torch.nn.Parameter) else None
            if target is not None and (target.data_ptr() % 16 != 0 or not target.is_contiguous()):
                target = None
            dpe = target if target is not None else torch.zeros((R, 64), dtype=torch.float32, device=dev)

            def table_grad():
                K.gemm(dQP, qv, dpe, M=R, N=64, K=chunk, a_mn=True, a_ld=R, b_mn=True, b_ld=q_ld, c_ld=64, nb1=H, nb2=S,
                       a_bs=(rows * R, chunk * R), b_bs=(64, chunk * q_ld), c_bs=(0, 0), alpha=scale, accumulate=2)
            if target is not None:
                _off_critical_path(table_grad, dQP, q_buf)
            else:
                table_grad()
            return dq_buf, None, (None if target is not None else dpe), None, None
        dQP = torch.empty((B, H, Tq, R), dtype=torch.bfloat16, device=dev)
        K.attn_dqp_scatter(dS, dQP, B, H, Tq, Tk, p_ld, maxpos)
        qpbs = (Tq * R, H * Tq * R)
        # dQ += scale dQP PE
        K.gemm(dQP, pe_hi, dqv, M=Tq, N=64, K=R, a_ld=R, b_mn=True, b_ld=64, c_ld=q_ld, nb1=H, nb2=B, a_bs=qpbs,
               b_bs=(0, 0), c_bs=(64, q_bs), alpha=scale, residual=dqv)
        # dPE[r,c] = scale sum_{b,h,i} dQP[b,h,i,r] q[b,i,h,c]
        parts = torch.empty((B * H, R * 64), dtype=torch.float32, device=dev)
        K.gemm(dQP, qv, parts, M=R, N=64, K=Tq, a_mn=True, a_ld=R, b_mn=True, b_ld=q_ld, c_ld=64, nb1=H, nb2=B,
               a_bs=qpbs, b_bs=(64, q_bs), c_bs=(R * 64, H * R * 64), alpha=scale)
        dpe = torch.empty((R, 64), dtype=torch.float32, device=dev)
        K.colsum(parts, dpe.view(-1))
        return dq_buf, None, dpe, None, None

    @staticmethod
    def _views(q_buf, kvb, cfg):
        d = cfg["d"]
        return (q_buf.narrow(2, cfg["q_col"] * d, d), kvb.narrow(2, cfg["k_col"] * d, d),
                kvb.narrow(2, cfg["v_col"] * d, d))

    @staticmethod
    def forward(ctx, q_buf, kv_buf, pe_k, key_pad, cfg):
        ctx.set_materialize_grads(False)
        same = kv_buf is None
        kvb = q_buf if same else kv_buf
        B, Tq, Tk = q_buf.shape[0], q_buf.shape[1], kvb.shape[1]
        H, d, scale = cfg["H"], cfg["d"], cfg["scale"]
        dev = q_buf.device
        p_ld = _pad8(Tk)
        qv, kk, vv = AttentionTCFn._views(q_buf, kvb, cfg)
        q_ld, q_bs, kv_ld, kv_bs = q_buf.stride(1), q_buf.stride(0), kvb.stride(1), kvb.stride(0)
        pbs = (Tq * p_ld, H * Tq * p_ld)
        maxpos = cfg.get("maxpos", 0)
        use_fused = RT.attn_fused and RT.attn_fused_bwd
        causal = bool(cfg.get("causal", False))
        rpe_fused = (pe_k is not None and use_fused and not causal and 0 < maxpos <= 160
                     and Tq <= maxpos and Tk <= maxpos and pe_k.shape[0] == 2 * maxpos)
        resident = rpe_fused or (pe_k is None and Tk <= 320 and use_fused)  # bounded score rows: one launch
        # streaming kernel (attention_flash.cu): any length, clipped relative positions; RT.attn_flash == "all" also
        # routes the shapes the resident kernel could take through it
        flash = (use_fused and RT.attn_flash and (pe_k is None or (not causal and maxpos > 0 and pe_k.shape[0] == 2 * maxpos))
                 and (not resident or RT.attn_flash == "all"))
        if resident or flash:
            # ONE launch: QK^T (+ the relative-position bias gathered on chip from QP = Q PE^T) -> masks ->
            # softmax -> dropout -> PV with the scores on chip. For the backward pass the kernel saves the
            # exponentials (bf16, dropout decision in the sign bit) and 1/rowsum; normalised fp32 probabilities are
            # written only when the caller asked for them (need_head_weights)
            drop_p = cfg.get("drop_p", 0.0)
            off = RT.next_offset() if drop_p > 0 else 0
            kp = _key_pad_u8(key_pad)
            want = bool(cfg.get("return_probs"))
            with_pe = pe_k is not None
            pe_hi = _pe_bf16(pe_k) if with_pe else None
            probs = torch.empty((B, H, Tq, p_ld), dtype=torch.float32, device=dev) if want else None
            # (inference: nothing is saved, the kernel skips those stores. needs_input_grad alone is not enough: under
            # torch.no_grad it still reports the relative-position table, a parameter)
            grad = cfg.get("grad_enabled", True) and any(ctx.needs_input_grad[:3])
            psave = torch.empty((B, H, Tq, p_ld), dtype=torch.bfloat16, device=dev) if grad else None
            inv_l = torch.empty((B, H, Tq), dtype=torch.float32, device=dev) if grad else None
            o32 = torch.empty((B, Tq, d), dtype=torch.float32, device=dev) if grad else None
            out = torch.empty((B, Tq, d), dtype=torch.bfloat16, device=dev)
            a = K.attn_args(B=B, H=H, Tq=Tq, Tk=Tk, dtype=K.dtype_id(q_buf), causal=int(cfg.get("causal", False)),
                            maxpos=maxpos if with_pe else 0, probs_dtype=K.dtype_id(probs) if want else 0, q=qv,
                            q_ld=q_ld, q_bs=q_bs, k=kk, k_ld=kv_ld, k_bs=kv_bs, v=vv, v_ld=kv_ld, v_bs=kv_bs,
                            key_pad=kp, pe_k=pe_hi, out=out, o_ld=d, o_bs=Tq * d, probs=probs, p_ld=p_ld, scale=scale,
                            drop_p=drop_p, seed=RT.seed, offset=off, probs_heads=cfg.get("probs_read_heads", 0) if want else 0)
            (K.attn_flash_fwd if flash else K.attn_fused_fwd)(a, None, psave, inv_l, o32)
            # `out` is an OUTPUT of this Function: it goes through save_for_backward (as an attribute of ctx it closes
            # the cycle out -> grad_fn -> ctx -> out, and psave / o32 of every layer would live until the next pass of
            # Python's cycle collector -- ~12 GB per eager update of the Large pre-training step)
            ctx.save_for_backward(q_buf, kv_buf, pe_k, probs, out)
            ctx.fused = (psave, inv_l, o32, kp)
            ctx.meta = (cfg, off, RT.seed, p_ld, same, pe_hi)
            cfg["_ext_ok"] = True  # this call's backward reads an external dP through the first probs_grad_heads heads only
            if probs is None:
                return out, None
            return out, probs[..., :Tk] if p_ld != Tk else probs
        S = torch.empty((B, H, Tq, p_ld), dtype=torch.float32, device=dev)
        K.gemm(qv, kk, S, M=Tq, N=Tk, K=64, a_ld=q_ld, b_ld=kv_ld, c_ld=p_ld, nb1=H, nb2=B, a_bs=(64, q_bs),
               b_bs=(64, kv_bs), c_bs=pbs, alpha=scale)
        QP, pe_hi, R = None, None, 0
        if pe_k is not None:
            R = pe_k.shape[0]
            pe_hi = _pe_bf16(pe_k)
            QP = torch.empty((B, H, Tq, R), dtype=torch.float32, device=dev)
            K.gemm(qv, pe_hi, QP, M=Tq, N=R, K=64, a_ld=q_ld, b_ld=64, c_ld=R, nb1=H, nb2=B, a_bs=(64, q_bs),
                   b_bs=(0, 0), c_bs=(Tq * R, H * Tq * R), alpha=scale)
        drop_p = cfg.get("drop_p", 0.0)
        off = RT.next_offset() if drop_p > 0 else 0
        kp = _key_pad_u8(key_pad)
        P = torch.empty((B, H, Tq, p_ld), dtype=torch.bfloat16, device=dev)
        Pd = torch.empty_like(P) if drop_p > 0 else None
        want = bool(cfg.get("return_probs"))
        K.attn_softmax_fwd(S, QP, kp, P, S if want else None, Pd, B, H, Tq, Tk, p_ld, cfg.get("causal", False),
                           cfg.get("maxpos", 0), drop_p, RT.seed, off)
        out = torch.empty((B, Tq, d), dtype=torch.bfloat16, device=dev)
        K.gemm(Pd if Pd is not None else P, vv, out, M=Tq, N=64, K=Tk, a_ld=p_ld, b_mn=True, b_ld=kv_ld, c_ld=d,
               nb1=H, nb2=B, a_bs=pbs, b_bs=(64, kv_bs), c_bs=(64, Tq * d))
        ctx.save_for_backward(q_buf, kv_buf, pe_k, P)
        ctx.meta = (cfg, off, RT.seed, p_ld, same, pe_hi)
        probs = S if want else P
        return out, probs[..., :Tk] if p_ld != Tk else probs

    @staticmethod
    def backward(ctx, dout, dprobs):
        q_buf, kv_buf, pe_k, P = ctx.saved_tensors[:4]
        cfg, off, seed, p_ld, same, pe_hi = ctx.meta
        fused = getattr(ctx, "fused", None)
        if fused is not None:
            fused = (ctx.saved_tensors[4],) + tuple(fused)  # (out, psave, inv_l, o32, key_pad)
        if fused is not None and pe_k is not None:
            return AttentionTCFn._fused_backward_rpe(q_buf, pe_k, pe_hi, cfg, off, seed, p_ld, fused, dout, dprobs)
        if fused is not None:
            return AttentionTCFn._fused_backward(q_buf, kv_buf, P, cfg, off, seed, p_ld, same, fused, dout, dprobs)
        if P.dtype != torch.bfloat16:  # fused forward returned fp32 probabilities to the caller
            P = P.to(torch.bfloat16)
        kvb = q_buf if same else kv_buf
        B, Tq, Tk = q_buf.shape[0], q_buf.shape[1], kvb.shape[1]
        H, d, scale = cfg["H"], cfg["d"], cfg["scale"]
        dev = q_buf.device
        drop_p = cfg.get("drop_p", 0.0)
        if dout is None:
            dout = torch.zeros((B, Tq, d), dtype=torch.bfloat16, device=dev)
        dout = dout.contiguous()
        qv, kk, vv = AttentionTCFn._views(q_buf, kvb, cfg)
        q_ld, q_bs, kv_ld, kv_bs = q_buf.stride(1), q_buf.stride(0), kvb.stride(1), kvb.stride(0)
        pbs = (Tq * p_ld, H * Tq * p_ld)
        full = q_buf.shape[2] == (3 * d if same else d)
        dq_buf = torch.empty_like(q_buf) if full else torch.zeros_like(q_buf)
        dkv_buf = dq_buf if same else torch.empty_like(kv_buf)
        dqv, dkk, dvv = AttentionTCFn._views(dq_buf, dkv_buf, cfg)
        # dP = dO V^T
        dP = torch.empty((B, H, Tq, p_ld), dtype=torch.float32, device=dev)
        K.gemm(dout, vv, dP, M=Tq, N=Tk, K=64, a_ld=d, b_ld=kv_ld, c_ld=p_ld, nb1=H, nb2=B, a_bs=(64, Tq * d),
               b_bs=(64, kv_bs), c_bs=pbs)
        dpx = None
        if dprobs is not None:
            dpx = dprobs
            if dpx.dtype != torch.float32 or dpx.shape[-1] != p_ld or not dpx.is_contiguous():
                buf = torch.zeros((B, H, Tq, p_ld), dtype=torch.float32, device=dev)
                buf[..., :Tk] = dprobs
                dpx = buf
        dS = torch.empty((B, H, Tq, p_ld), dtype=torch.bfloat16, device=dev)
        Pd = torch.empty_like(P) if drop_p > 0 else None
        K.attn_ds(P, dP, dpx, dS, Pd, B, H, Tq, Tk, p_ld, drop_p, seed, off)
        if Pd is None:
            Pd = P
        # dV[j,c] = sum_i Pd[i,j] dO[i,c]   (both operands MN-major: no transposes)
        K.gemm(Pd, dout, dvv, M=Tk, N=64, K=Tq, a_mn=True, a_ld=p_ld, b_mn=True, b_ld=d, c_ld=kv_ld, nb1=H, nb2=B,
               a_bs=pbs, b_bs=(64, Tq * d), c_bs=(64, kv_bs))
        # dQ = scale dS K ; dK = scale dS^T Q
        K.gemm(dS, kk, dqv, M=Tq, N=64, K=Tk, a_ld=p_ld, b_mn=True, b_ld=kv_ld, c_ld=q_ld, nb1=H, nb2=B, a_bs=pbs,
               b_bs=(64, kv_bs), c_bs=(64, q_bs), alpha=scale)
        K.gemm(dS, qv, dkk, M=Tk, N=64, K=Tq, a_mn=True, a_ld=p_ld, b_mn=True, b_ld=q_ld, c_ld=kv_ld, nb1=H, nb2=B,
               a_bs=pbs, b_bs=(64, q_bs), c_bs=(64, kv_bs), alpha=scale)
        dpe = None
        if pe_k is not None:
            R = pe_k.shape[0]
            dQP = torch.empty((B, H, Tq, R), dtype=torch.bfloat16, device=dev)
            K.attn_dqp_scatter(dS, dQP, B, H, Tq, Tk, p_ld, cfg.get("maxpos", 0))
            qpbs = (Tq * R, H * Tq * R)
            # dQ += scale dQP PE
            K.gemm(dQP, pe_hi, dqv, M=Tq, N=64, K=R, a_ld=R, b_mn=True, b_ld=64, c_ld=q_ld, nb1=H, nb2=B, a_bs=qpbs,
                   b_bs=(0, 0), c_bs=(64, q_bs), alpha=scale, residual=dqv)
            # dPE[r,c] = scale sum_{b,h,i} dQP[b,h,i,r] q[b,i,h,c]
            parts = torch.empty((B, H, R, 64), dtype=torch.float32, device=dev)
            K.gemm(dQP, qv, parts, M=R, N=64, K=Tq, a_mn=True, a_ld=R, b_mn=True, b_ld=q_ld, c_ld=64, nb1=H, nb2=B,
                   a_bs=qpbs, b_bs=(64, q_bs), c_bs=(R * 64, H * R * 64), alpha=scale)
            dpe = parts.sum(dim=(0, 1))
        return dq_buf, (None if same else dkv_buf), dpe, None, None


def attention_decode(q_buf, kv_buf, *, H, d, q_col, k_col, v_col, scale, key_pad=None, return_probs=False,
                     kv_rows=None, kv_div=1):
    """One query row per utterance (incremental decoding, forward only) on st5_attn_decode_fwd: q_buf [B, 1, nq*d],
    kv_buf [B, Tk, nk*d] with q / k / v in column blocks q_col / k_col / v_col (kv_buf None: q_buf), key_pad [B, Tk]
    (nonzero / True = masked). Returns (out [B, 1, d], probs [B, H, 1, Tk] fp32 when return_probs else None).
    Beam search (st5_attn_lineage_fwd, no probabilities): kv_rows int32 [B, >= Tk] names the kv_buf row of each key of
    query row b, or kv_div > 1 makes query row b read kv_buf row b // kv_div."""
    kvb = q_buf if kv_buf is None else kv_buf
    B, Tk = q_buf.shape[0], kvb.shape[1]
    hd = d // H  # (64: st5_attn_decode_fwd / st5_attn_lineage_fwd; 80: their st5_*_hd_fwd counterparts)
    assert q_buf.shape[1] == 1 and d == H * hd and hd in (64, 80) and q_buf.dtype == kvb.dtype
    wide = {} if hd == 64 else dict(head_dim=hd)
    if kv_rows is not None or kv_div != 1:
        assert not return_probs
        out = torch.empty((B, 1, d), dtype=q_buf.dtype, device=q_buf.device)
        (K.attn_lineage_fwd if hd == 64 else K.attn_lineage_hd_fwd)(
            q_buf.narrow(2, q_col * d, d), kvb.narrow(2, k_col * d, d), kvb.narrow(2, v_col * d, d), out,
            H=H, scale=scale, key_pad=_key_pad_u8(key_pad), kv_rows=kv_rows, kv_div=kv_div, **wide)
        return out, None
    assert kvb.shape[0] == B
    out = torch.empty((B, 1, d), dtype=q_buf.dtype, device=q_buf.device)
    probs = torch.empty((B, H, 1, Tk), dtype=torch.float32, device=q_buf.device) if return_probs else None
    (K.attn_decode_fwd if hd == 64 else K.attn_decode_hd_fwd)(
        q_buf.narrow(2, q_col * d, d), kvb.narrow(2, k_col * d, d), kvb.narrow(2, v_col * d, d), out,
        H=H, scale=scale, key_pad=_key_pad_u8(key_pad), probs=probs, **wide)
    return out, probs


def attention_rows(q_buf, kv_buf, *, H, d, q_col, k_col, v_col, scale, key_pad=None, causal=False):
    """Forward-only attention for heads the fused kernels do not take (80 channels): every query row of q_buf [B, Tq, *]
    becomes one row of the one-row kernel over its utterance's keys (kv_div = Tq), with the causal mask and key_pad folded
    into one [B*Tq, Tk] key mask. Returns (out [B, Tq, d], None)."""
    if torch.is_grad_enabled() and (q_buf.requires_grad or (kv_buf is not None and kv_buf.requires_grad)):
        raise NotImplementedError(f"attention over heads of {d // H} channels is forward-only (the fused attention "
                                  "kernels and their backward take 64)")
    kvb = q_buf if kv_buf is None else kv_buf
    B, Tq, Tk = q_buf.shape[0], q_buf.shape[1], kvb.shape[1]
    mask = torch.zeros((B, Tq, Tk), dtype=torch.bool, device=q_buf.device)
    if causal:
        mask |= torch.ones((Tq, Tk), dtype=torch.bool, device=q_buf.device).triu(1)
    if key_pad is not None:
        mask |= key_pad.bool()[:, None, :]
    q_rows = q_buf.contiguous().view(B * Tq, 1, q_buf.shape[2])
    out, _ = attention_decode(q_rows, kvb, H=H, d=d, q_col=q_col, k_col=k_col, v_col=v_col, scale=scale,
                              key_pad=mask.view(B * Tq, Tk), kv_div=Tq)
    return out.view(B, Tq, d), None


def attention(q_buf, kv_buf, *, H, d, q_col, k_col, v_col, scale, pe_k=None, maxpos=0, key_pad=None, causal=False,
              drop_p=0.0, return_probs=False):
    if RT.attn_decode_rows and q_buf.shape[1] == 1 and pe_k is None and not causal and drop_p == 0.0 \
            and not torch.is_grad_enabled():
        return attention_decode(q_buf, kv_buf, H=H, d=d, q_col=q_col, k_col=k_col, v_col=v_col, scale=scale,
                                key_pad=key_pad, return_probs=return_probs)
    if d != H * 64:  # (80-channel heads: forward only, on the one-row kernel)
        assert pe_k is None and drop_p == 0.0 and not return_probs
        return attention_rows(q_buf, kv_buf, H=H, d=d, q_col=q_col, k_col=k_col, v_col=v_col, scale=scale,
                              key_pad=key_pad, causal=causal)
    # RT.probs_grad_heads: the consumer of the returned probabilities differentiates only through the first n heads (the
    # guided-attention loss; set by the trainer from the criterion): the backward skips the zero gradient of the others
    cfg = dict(H=H, d=d, q_col=q_col, k_col=k_col, v_col=v_col, scale=scale, maxpos=maxpos, causal=causal,
               drop_p=drop_p, return_probs=return_probs, probs_grad_heads=RT.probs_grad_heads if return_probs else 0,
               probs_read_heads=RT.probs_read_heads if return_probs else 0, grad_enabled=torch.is_grad_enabled())
    Tk = (q_buf if kv_buf is None else kv_buf).shape[1]
    streaming = RT.attn_flash and RT.attn_fused and RT.attn_fused_bwd and (pe_k is None or not causal)
    if q_buf.dtype == torch.bfloat16 and RT.attn_tensor_core and (Tk <= 512 or streaming):
        out, probs = AttentionTCFn.apply(q_buf, kv_buf, pe_k, key_pad, cfg)
        if probs is not None and cfg.get("_ext_ok") and cfg["probs_grad_heads"] > 0:
            # tells a producer of dP (criterions.text_to_speech_loss.GuidedAttnFn) that heads >= n are never read: it
            # may leave them unwritten instead of clearing 10 of 12 heads of a [B,H,Tq,Tk] fp32 tensor
            probs._st5_ext_heads = cfg["probs_grad_heads"]
        return out, probs
    return AttentionFn.apply(q_buf, kv_buf, pe_k, key_pad, cfg)


# =================================================================================================== postnet blocks
def _conv_wgrad_split(Cout, Ncols, Kd):
    """Split of the post-net weight-gradient contraction (K = all frames of the batch, ~20 k) over the GEMM's batch
    dimension: (S, chunk) with S * chunk >= Kd, chunk a multiple of 8 rows. The output has a handful of 128 x 128 tiles
    only, so without the split a few CTAs would do all the work; S fills one wave of the 132 SMs."""
    tiles = ((Cout + 127) // 128) * ((Ncols + 127) // 128)
    S = max(1, min(32, 132 // max(1, tiles), Kd // 512))
    chunk = ((Kd + S - 1) // S + 7) // 8 * 8
    return S, chunk


class Conv1dK5Fn(torch.autograd.Function):
    """Conv1d(kernel 5, padding 2, no bias) on channels-last activations [B,T,Cin] as ONE GEMM over an
    overlapping-window view of the zero-padded buffer (no im2col): out[b,t,:] = W2 . xpad[b, t:t+5, :].ravel().
    espnet Postnet convs behind speech_decoder_postnet.py:39-51."""

    @staticmethod
    def forward(ctx, x, weight):
        B, T, Cin = x.shape
        Cout, _, Kw = weight.shape
        pad = (Kw - 1) // 2
        Tp = T + 2 * pad
        # (zero rows past the batch: the split weight-gradient GEMM of the backward reads whole chunks)
        S, chunk = _conv_wgrad_split(Cout, Kw * Cin, B * Tp - 2 * pad)
        rows = max(B * Tp, S * chunk + 2 * pad)
        xflat = torch.zeros((rows, Cin), dtype=x.dtype, device=x.device)
        xp = xflat[:B * Tp].view(B, Tp, Cin)
        xp[:, pad:pad + T] = x
        w_sh = RT.shadow(("conv_f", id(weight)), lambda: weight.detach().permute(0, 2, 1).reshape(Cout, Kw * Cin))
        ldc = _pad8(Cout)
        out = torch.empty((B, T, ldc), dtype=x.dtype, device=x.device)
        xa = _split(xflat)
        # window GEMM: rows t (per batch b), K = Kw*Cin contiguous starting at xpad[b, t]; ld = Cin
        _conv_mm(xa, w_sh, out, B=B, T=T, Tp=Tp, Cin=Cin, Cout=Cout, Kw=Kw, ldc=ldc)
        ctx.save_for_backward(weight)
        ctx.xa = xa
        ctx.meta = (B, T, Tp, Cin, Cout, Kw, pad)
        return out if ldc == Cout else out[..., :Cout]

    @staticmethod
    def backward(ctx, dy):
        (weight,) = ctx.saved_tensors
        B, T, Tp, Cin, Cout, Kw, pad = ctx.meta
        dev = dy.device
        Kd = B * Tp - 2 * pad
        S, chunk = _conv_wgrad_split(Cout, Kw * Cin, Kd)
        rows = max(B * Tp, S * chunk + 2 * pad)
        dflat = torch.zeros((rows, Cout), dtype=dy.dtype, device=dev)
        dyp = dflat[:B * Tp].view(B, Tp, Cout)
        dyp[:, pad:pad + T] = dy
        ga = _split(dflat)
        # dx[b,t,ci] = sum_{u,co} dypad[b,t+u,co] * W[co,ci,Kw-1-u]
        w_b = RT.shadow(("conv_b", id(weight)),
                        lambda: weight.detach().flip(2).permute(1, 2, 0).reshape(Cin, Kw * Cout))
        ldx = _pad8(Cin)
        dx = torch.empty((B, T, ldx), dtype=dy.dtype, device=dev)
        _conv_mm(ga, w_b, dx, B=B, T=T, Tp=Tp, Cin=Cout, Cout=Cin, Kw=Kw, ldc=ldx)
        # dW2[co, u*Cin+ci] = sum_rho dypad_flat[rho+pad, co] * xpad_flat[rho+u, ci]  (both MN-major, K = B*Tp - 2*pad)
        a_ops = tuple(None if t is None else t[pad:] for t in ga)
        if ga[1] is None and ctx.xa[1] is None and RT.wgrad_splitk and S > 1 and Cout % 8 == 0 and Cin % 8 == 0:
            # contraction split over the batch dimension, partial products added at the L2 (st5_gemm_bf16 accumulate 2);
            # rows past Kd are the zero tails of both buffers
            dW2 = torch.zeros((Cout, Kw * Cin), dtype=torch.float32, device=dev)
            K.gemm(a_ops[0], ctx.xa[0], dW2, M=Cout, N=Kw * Cin, K=chunk, a_mn=True, a_ld=Cout, b_mn=True, b_ld=Cin,
                   c_ld=Kw * Cin, nb1=S, nb2=1, a_bs=(chunk * Cout, 0), b_bs=(chunk * Cin, 0), c_bs=(0, 0), accumulate=2)
        else:
            dW2 = torch.empty((Cout, Kw * Cin), dtype=torch.float32, device=dev)
            mm(a_ops, ctx.xa, dW2, M=Cout, N=Kw * Cin, Kd=Kd, a_mn=True, a_ld=Cout, b_mn=True, b_ld=Cin, c_ld=Kw * Cin)
        dW = dW2.view(Cout, Kw, Cin).permute(0, 2, 1).contiguous()
        ctx.xa = None
        return (dx if ldx == Cin else dx[..., :Cin]), dW


def _conv_mm(xa, w_sh, out, *, B, T, Tp, Cin, Cout, Kw, ldc):
    """Batched window GEMM used by Conv1dK5Fn (fwd and dgrad). xa = (hi, lo) of the padded [B*Tp, Cin] buffer."""
    a_hi, a_lo = xa
    b_hi, b_lo = w_sh
    kw = dict(M=T, N=Cout, K=Kw * Cin, a_ld=Cin, b_ld=Kw * Cin, c_ld=ldc, nb1=B, nb2=1, a_bs=(Tp * Cin, 0),
              b_bs=(0, 0), c_bs=(T * ldc, 0))
    if a_lo is None:
        K.gemm(a_hi, b_hi, out, **kw)
        return
    K.gemm(a_hi, b_hi, out, **kw)
    K.gemm(a_hi, b_lo, out, accumulate=True, **kw)
    K.gemm(a_lo, b_hi, out, accumulate=True, **kw)


def conv1d_k5(x, weight):
    return Conv1dK5Fn.apply(x, weight)


class BatchNormActFn(torch.autograd.Function):
    """dropout(act(BatchNorm1d(x))) on channels-last rows; training statistics over all B*T rows."""

    @staticmethod
    def forward(ctx, x, gamma, beta, running_mean, running_var, training, momentum, eps, act, drop_p):
        x = x.contiguous()
        Cc = x.shape[-1]
        rows = x.numel() // Cc
        dev = x.device
        y = torch.empty_like(x)
        y_pre = torch.empty_like(x) if act is not None else None
        mean = torch.empty(Cc, dtype=torch.float32, device=dev)
        rstd = torch.empty_like(mean)
        scratch = torch.empty(2 * Cc, dtype=torch.float32, device=dev)
        off = RT.next_offset() if drop_p > 0 else 0
        K.bn_fwd(x, Cc, gamma.detach(), beta.detach(), running_mean, running_var, mean, rstd, y, Cc, y_pre, rows, Cc,
                 training, momentum, eps, act, drop_p, RT.seed, off, scratch)
        ctx.save_for_backward(x, y_pre, gamma, mean, rstd)
        ctx.meta = (act, drop_p, off, RT.seed, rows, Cc, training)
        ctx.param_ids = (id(gamma), id(beta))
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y_pre, gamma, mean, rstd = ctx.saved_tensors
        act, drop_p, off, seed, rows, Cc, training = ctx.meta
        if not training:
            raise RuntimeError("BatchNormActFn backward is only defined for training-mode statistics")
        dy = dy.contiguous()
        dx = torch.empty_like(dy)
        # the kernel ADDS the parameter gradients: aim it at the trainer's flat gradient buffer when one is registered
        # (like ResidualLayerNormFn: no zero fills, no AccumulateGrad adds), else at fresh zero vectors for autograd
        gid, bid = ctx.param_ids
        gG, gB = RT._static_grad.get(("bias", gid)), RT._static_grad.get(("bias", bid))
        direct = gG is not None and gB is not None
        dgamma = gG if direct else torch.zeros(Cc, dtype=torch.float32, device=dy.device)
        dbeta = gB if direct else torch.zeros(Cc, dtype=torch.float32, device=dy.device)
        scratch = torch.empty(2 * Cc, dtype=torch.float32, device=dy.device)
        K.bn_bwd(dy, Cc, x, Cc, y_pre, gamma.detach(), mean, rstd, dx, Cc, dgamma, dbeta, rows, Cc, act, drop_p, seed,
                 off, scratch)
        if direct:
            dgamma = dbeta = None
        return dx, dgamma, dbeta, None, None, None, None, None, None, None


def batch_norm_act(x, bn, training, act=None, drop_p=0.0):
    if training and bn.num_batches_tracked is not None:
        bn.num_batches_tracked += 1  # torch.nn.BatchNorm1d bookkeeping (checkpoint parity)
    return BatchNormActFn.apply(x, bn.weight, bn.bias, bn.running_mean, bn.running_var, training,
                                bn.momentum if bn.momentum is not None else 0.1, bn.eps, act, drop_p)


class DropoutFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, drop_p):
        x = x.contiguous()
        y = torch.empty_like(x)
        off = RT.next_offset()
        K.dropout(x, y, drop_p, RT.seed, off)
        ctx.meta = (drop_p, off, RT.seed)
        return y

    @staticmethod
    def backward(ctx, dy):
        drop_p, off, seed = ctx.meta
        dy = dy.contiguous()
        dx = torch.empty_like(dy)
        K.dropout(dy, dx, drop_p, seed, off)
        return dx, None


def dropout(x, drop_p, training=True):
    if drop_p <= 0.0 or not training:
        return x
    return DropoutFn.apply(x, drop_p)


# =================================================================================================== speaker head
def _operands(x):
    """fp32 [rows, cols] (unit inner stride) -> GEMM operands in padded rows: the (hi, lo) bf16 split in parity mode,
    (hi, None) in throughput mode."""
    rows, cols = x.shape
    pair = torch.empty((2 if RT.dtype == torch.float32 else 1, rows, _pad8(cols)), dtype=torch.bfloat16, device=x.device)
    hi = pair[0, :, :cols]
    lo = pair[1, :, :cols] if pair.shape[0] == 2 else None
    K.cast_bf16(x, hi, lo)
    return hi, lo


def _padded_f32(t):
    """fp32 view with unit inner stride and a 16-byte aligned row pitch (what the GEMM and row kernels read)."""
    t = t.float()
    if t.stride(1) == 1 and t.stride(0) % 8 == 0 and t.data_ptr() % 16 == 0:
        return t
    buf = torch.empty((t.shape[0], _pad8(t.shape[1])), dtype=torch.float32, device=t.device)[:, :t.shape[1]]
    buf.copy_(t)
    return buf


class L2NormRowsFn(torch.autograd.Function):
    """F.normalize(x, p=2, dim=1) (speaker_decoder_postnet.py:190-191) -> fp32 rows. grad_key: the trainer's flat
    gradient view the input gradient is accumulated into (the class weight), if one is registered."""

    @staticmethod
    def forward(ctx, x, grad_key):
        x2 = x if x.stride(-1) == 1 else x.contiguous()
        y = torch.empty(x2.shape, dtype=torch.float32, device=x.device)
        nrm = torch.empty(x2.shape[0], dtype=torch.float32, device=x.device)
        K.l2norm_rows_fwd(x2, y, nrm)
        ctx.save_for_backward(y, nrm)
        ctx.meta = (x.dtype, grad_key)
        return y

    @staticmethod
    def backward(ctx, dy):
        y, nrm = ctx.saved_tensors
        dtype, grad_key = ctx.meta
        dy = dy.float().contiguous()
        target = RT._static_grad.get(grad_key) if grad_key is not None else None
        if target is not None:
            K.l2norm_rows_bwd(dy, y, nrm, target, accumulate=True)
            return None, None
        dx = torch.empty(y.shape, dtype=dtype, device=y.device)
        K.l2norm_rows_bwd(dy, y, nrm, dx)
        return dx, None


def l2_normalize_rows(x, grad_key=None):
    return L2NormRowsFn.apply(x, grad_key)


class CosineFn(torch.autograd.Function):
    """out [B, N] fp32 = xn . wn^T (F.linear(x_norm, w_norm), speaker_decoder_postnet.py:192) and its two gradient
    GEMMs on the wgmma kernel; parity mode contracts the hi/lo splits."""

    @staticmethod
    def forward(ctx, xn, wn):
        B, E = xn.shape
        N = wn.shape[0]
        ldc = _pad8(N)
        out = torch.empty((B, ldc), dtype=torch.float32, device=xn.device)
        xa, wa = _operands(xn), _operands(wn)
        mm(xa, wa, out, M=B, N=N, Kd=E, a_ld=xa[0].stride(0), b_ld=wa[0].stride(0), c_ld=ldc)
        ctx.ops = (xa, wa)
        return out[:, :N]

    @staticmethod
    def backward(ctx, dc):
        xa, wa = ctx.ops
        B, E = xa[0].shape
        N = wa[0].shape[0]
        ga = _operands(_padded_f32(dc))
        dxn = dwn = None
        if ctx.needs_input_grad[0]:
            dxn = torch.empty((B, E), dtype=torch.float32, device=dc.device)
            mm(ga, wa, dxn, M=B, N=E, Kd=N, a_ld=ga[0].stride(0), b_mn=True, b_ld=wa[0].stride(0), c_ld=E)
        if ctx.needs_input_grad[1]:
            dwn = torch.empty((N, E), dtype=torch.float32, device=dc.device)
            mm(ga, xa, dwn, M=N, N=E, Kd=B, a_mn=True, a_ld=ga[0].stride(0), b_mn=True, b_ld=xa[0].stride(0), c_ld=E)
        return dxn, dwn


def cosine(xn, wn):
    return CosineFn.apply(xn, wn)


class MarginFn(torch.autograd.Function):
    """AngularMargin / AdditiveAngularMargin (speaker_decoder_postnet.py:48-126) on the cosines with the margin on
    column mtarget[b] of row b; margin = (mode, scale, m, easy_margin)."""

    @staticmethod
    def forward(ctx, cos, mtarget, margin):
        cos = _padded_f32(cos)
        B, N = cos.shape
        z = torch.empty((B, _pad8(N)), dtype=torch.float32, device=cos.device)[:, :N]
        K.margin_ce_fwd(cos, mtarget, margin, z_out=z)
        ctx.save_for_backward(cos, mtarget)
        ctx.margin = margin
        return z

    @staticmethod
    def backward(ctx, dz):
        cos, mtarget = ctx.saved_tensors
        B, N = cos.shape
        dx = torch.empty((B, _pad8(N)), dtype=torch.float32, device=cos.device)[:, :N]
        K.margin_ce_bwd(cos, mtarget, ctx.margin, dx, dz=_padded_f32(dz))
        return dx, None, None


def margin_logits(cos, mtarget, margin):
    return MarginFn.apply(cos, mtarget.contiguous(), margin)


class MarginCEFn(torch.autograd.Function):
    """Label-smoothed cross entropy of SpeechtoTextLoss on class logits [B, N] (speech_to_text_loss.py:93-110, 340-372)
    in one row kernel: returns the sums (loss, nll, n_correct, total) over the rows; only loss and nll carry gradient."""

    @staticmethod
    def forward(ctx, z, target, eps, ignore_index):
        z = _padded_f32(z)
        B, N = z.shape
        stats = torch.empty((B, 4), dtype=torch.float32, device=z.device)
        lse = torch.empty(B, dtype=torch.float32, device=z.device)
        target = target.reshape(-1).contiguous()
        K.margin_ce_fwd(z, None, None, target=target, eps=eps, ignore_index=ignore_index, stats=stats, lse=lse)
        sums = torch.empty(4, dtype=torch.float32, device=z.device)
        K.colsum(stats, sums)
        ctx.save_for_backward(z, target, lse)
        ctx.meta = (eps, ignore_index)
        return sums

    @staticmethod
    def backward(ctx, g):
        z, target, lse = ctx.saved_tensors
        eps, ignore_index = ctx.meta
        B, N = z.shape
        dz = torch.empty((B, _pad8(N)), dtype=torch.float32, device=z.device)[:, :N]
        K.margin_ce_bwd(z, None, None, dz, target=target, eps=eps, ignore_index=ignore_index, lse=lse,
                        gstat=g.float().contiguous())
        return dz, None, None, None


def margin_ce(z, target, eps, ignore_index):
    return MarginCEFn.apply(z, target, eps, ignore_index)


class TimeMeanFn(torch.autograd.Function):
    """x [B, T, C] -> mean over all T frames (padding included, models/speecht5.py:838)."""

    @staticmethod
    def forward(ctx, x):
        x = x.contiguous()
        B, T, Cc = x.shape
        y = torch.empty((B, Cc), dtype=x.dtype, device=x.device)
        K.time_mean_fwd(x, y)
        ctx.shape = x.shape
        return y

    @staticmethod
    def backward(ctx, dy):
        dx = torch.empty(ctx.shape, dtype=dy.dtype, device=dy.device)
        K.time_mean_bwd(dy.contiguous(), dx)
        return dx


def time_mean(x):
    return TimeMeanFn.apply(x)
