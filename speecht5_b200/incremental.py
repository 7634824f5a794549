"""Incremental decoding with a key/value cache (SURVEY section 8a row 21 / 8f-2; the reference keeps fairseq
incremental state: speecht5/models/modules/multihead_attention.py:255-330, transformer_layer.py:262-404,
decoder.py:171-269). Opt-in: `use_cache=True` on generate_speech / generate_text_greedy runs the step eagerly,
`use_cache="graph"` on generate_speech replays ONE captured CUDA graph per decoder step (SynthesisGraph below). Checked
on the CPU against the prefix-recomputing path through the kernel emulation (tests/test_frontend_cpu.py) and on the
device (tests/test_frontend_gpu.py); nothing on the training path imports this module.

Per utterance batch the cross-attention keys / values of every decoder layer are projected ONCE; every step projects
q | k | v of the single new row, appends k | v to the layer's [B, T_max, 2C] cache and attends over the cache with a
one-row query -- O(L) work per step instead of the O(L^2) prefix recomputation. All contractions run on the existing
GEMM, the one-row attention on the split-KV decode kernel (st5_attn_decode_fwd), which takes strided key / value
views."""
import torch

from . import kernels, ops
from .ops import RT


def _act_dtype(x):
    return x if x.dtype == RT.dtype else x.to(RT.dtype)


def _attend(*a, **kw):
    """One-row queries: the split-KV decode kernel (st5_attn_decode_fwd; the fused wgmma path works on 64-query tiles)."""
    prev = RT.attn_decode_rows
    RT.attn_decode_rows = True
    try:
        return ops.attention(*a, **kw)
    finally:
        RT.attn_decode_rows = prev


class DecoderCache:
    def __init__(self, decoder, encoder_out, max_len):
        enc = encoder_out.get("_encoder_out_btc")
        if enc is None:
            enc = encoder_out["encoder_out"][0].transpose(0, 1).contiguous()
        enc = _act_dtype(enc)
        pm = encoder_out["encoder_padding_mask"]
        self.enc_pad = pm[0] if len(pm) > 0 else None
        B, _, C = enc.shape
        self.t = 0
        self.max_len = max_len
        self.cross, self.self_kv = [], []
        for layer in decoder.layers:
            ca = layer.encoder_attn
            self.cross.append(ops.linear(enc, (ca.k_proj.weight, ca.v_proj.weight), (ca.k_proj.bias, ca.v_proj.bias)))
            self.self_kv.append(torch.zeros((B, max_len, 2 * C), dtype=RT.dtype, device=enc.device))

    def reorder(self, new_order):
        """decoder.reorder_incremental_state_scripting (beam reordering): select utterances along the batch axis."""
        self.cross = [c.index_select(0, new_order) for c in self.cross]
        self.self_kv = [c.index_select(0, new_order) for c in self.self_kv]
        if self.enc_pad is not None:
            self.enc_pad = self.enc_pad.index_select(0, new_order)


@torch.no_grad()
def decoder_step(decoder, x_new, cache, need_head_weights=False, t_dev=None, span=None, self_pad=None, self_rows=None,
                 cross_div=1):
    """x_new [B, 1, C] = decoder-prenet output of the newest position. Returns (x [B, 1, C], [attn [B, H, 1, S]] per
    layer or None). Evaluation semantics (no dropout, no LayerDrop) -- generation only.

    Device-side step index (the form a captured graph replays): `t_dev` int64 [1] holds the position, the new key / value
    row is written with index_copy_, and self-attention runs over the first `span` cache rows with `self_pad` (uint8
    [B, span], 1 = position > t) masking what has not been written yet -- no host scalar depends on the step.

    Beam search (BeamGraph, device-step form only): `self_rows` int32 [B, >= span] is the lineage table -- key j of row b
    is read from cache row self_rows[b, j] -- and with cross_div = K row b attends over cross keys / values row b // K
    (one copy per sentence). Neither returns attention probabilities."""
    assert not decoder.training
    x = _act_dtype(x_new).contiguous()
    t = cache.t
    assert t_dev is not None or t < cache.max_len
    attns = []
    for li, layer in enumerate(decoder.layers):
        sa, ca = layer.self_attn, layer.encoder_attn
        C = sa.embed_dim
        residual = x
        h = ops.residual_layer_norm(x, None, layer.self_attn_layer_norm) if layer.normalize_before else x
        qkv = ops.linear(h, (sa.q_proj.weight, sa.k_proj.weight, sa.v_proj.weight),
                         (sa.q_proj.bias, sa.k_proj.bias, sa.v_proj.bias))  # [B, 1, 3C]
        if t_dev is None:
            cache.self_kv[li][:, t] = qkv[:, 0, C:]
            a, _ = _attend(qkv, cache.self_kv[li][:, : t + 1], H=sa.num_heads, d=C, q_col=0, k_col=0, v_col=1,
                           scale=sa.scaling)
        elif self_rows is not None:
            cache.self_kv[li].index_copy_(1, t_dev, qkv[:, :, C:])
            a, _ = ops.attention_decode(qkv, cache.self_kv[li][:, :span], H=sa.num_heads, d=C, q_col=0, k_col=0, v_col=1,
                                        scale=sa.scaling, key_pad=self_pad, kv_rows=self_rows)
        else:
            cache.self_kv[li].index_copy_(1, t_dev, qkv[:, :, C:])
            a, _ = _attend(qkv, cache.self_kv[li][:, :span], H=sa.num_heads, d=C, q_col=0, k_col=0, v_col=1,
                           scale=sa.scaling, key_pad=self_pad)
        if layer.normalize_before:
            x = ops.linear(a, sa.out_proj.weight, sa.out_proj.bias, residual=residual)
        else:
            x = ops.residual_layer_norm(ops.linear(a, sa.out_proj.weight, sa.out_proj.bias), residual,
                                        layer.self_attn_layer_norm)
        if ca is None:  # a decoder without encoder attention (the fusion LM, lm.TransformerLM): pre-LN only
            assert layer.normalize_before
            x = ops.ffn(ops.residual_layer_norm(x, None, layer.final_layer_norm), layer.fc1, layer.fc2,
                        layer.activation_fn, residual=x)
            continue
        residual = x
        h = ops.residual_layer_norm(x, None, layer.encoder_attn_layer_norm) if layer.normalize_before else x
        q = ops.linear(h, ca.q_proj.weight, ca.q_proj.bias)
        if cross_div != 1:
            a, probs = ops.attention_decode(q, cache.cross[li], H=ca.num_heads, d=C, q_col=0, k_col=0, v_col=1,
                                            scale=ca.scaling, key_pad=cache.enc_pad, kv_div=cross_div)
        else:
            a, probs = _attend(q, cache.cross[li], H=ca.num_heads, d=C, q_col=0, k_col=0, v_col=1, scale=ca.scaling,
                               key_pad=cache.enc_pad, return_probs=need_head_weights)
        if need_head_weights:
            attns.append(probs.float())
        if layer.normalize_before:
            x = ops.linear(a, ca.out_proj.weight, ca.out_proj.bias, residual=residual)
            x = ops.ffn(ops.residual_layer_norm(x, None, layer.final_layer_norm), layer.fc1, layer.fc2,
                        layer.activation_fn, residual=x)
        else:
            x = ops.residual_layer_norm(ops.linear(a, ca.out_proj.weight, ca.out_proj.bias), residual,
                                        layer.encoder_attn_layer_norm)
            x = ops.residual_layer_norm(ops.ffn(x, layer.fc1, layer.fc2, layer.activation_fn), x,
                                        layer.final_layer_norm)
    if decoder.layer_norm is not None:
        x = ops.residual_layer_norm(x, None, decoder.layer_norm)
    if t_dev is None:
        cache.t = t + 1
    return x, (attns if need_head_weights else None)


class _StaticCache:
    """DecoderCache with caller-owned, fixed-size buffers (a captured graph bakes their addresses)."""

    def __init__(self, cross, self_kv, enc_pad, max_len):
        self.cross, self.self_kv, self.enc_pad, self.max_len, self.t = cross, self_kv, enc_pad, max_len, 0


class SynthesisGraph:
    """Greedy speech synthesis (models/speecht5.py:1188-1249) of B utterances at once, with every decoder step = ONE
    CUDA-graph replay: prenet on each utterance's newest frame (always-on dropout drawn from the device-resident seed,
    advanced inside the graph), positional row gathered by the device step counter, the key/value-cached decoder,
    feat_out | prob_out, each utterance's stopping rule, and the step's outputs written into preallocated result buffers
    at the step index. B = 1 is generate_speech(use_cache="graph"); generate_speech_batch uses any B.

    The object is utterance-independent and is kept on the model (`synthesis_graph`): every buffer a graph reads has a
    fixed size -- the cross-attention keys / values of utterance b are copied into row b of [B, S_bucket, 2C] buffers
    with the tail masked, the frame budget is a bucket too -- so the graphs captured for one batch serve every later one
    of the same buckets (serving: no capture on the request path after the first). Self-attention spans are bucketed
    (128, 256, ...): one graph per span, so a step attends over at most 2x the keys it needs. Every row keeps the
    reference's stopping rule (:1235-1245) with its own minlen / maxlen; the done flags and lengths are device tensors
    written inside the graph. The host replays `chunk` steps, then reads their "all done" flags in one copy; rows that
    finished earlier keep running and what they compute past their length is discarded."""

    CHUNK = 8

    def __init__(self, model, S_bucket, maxlen_bucket, device, capture=True, B=1, attention=True):
        self.m = model
        self.capture = capture  # False: the same step body runs eagerly (CPU checks of the device-counter form)
        dec, post = model.decoder, model.speech_decoder_postnet
        dev = torch.device(device)
        self.dev, self.r, self.odim = dev, model.reduction_factor, post.odim
        self.B, self.S, self.maxlen = int(B), int(S_bucket), int(maxlen_bucket)
        B = self.B
        rows = self.maxlen + self.CHUNK
        L, H = len(dec.layers), dec.layers[0].encoder_attn.num_heads
        C = dec.layers[0].self_attn.embed_dim
        self.cache = _StaticCache([torch.zeros((B, self.S, 2 * C), dtype=RT.dtype, device=dev) for _ in dec.layers],
                                  [torch.zeros((B, rows, 2 * C), dtype=RT.dtype, device=dev) for _ in dec.layers],
                                  torch.zeros((B, self.S), dtype=torch.uint8, device=dev), rows)
        self.t = torch.zeros(1, dtype=torch.int64, device=dev)
        self.ys_last = torch.zeros(B, 1, self.odim, dtype=torch.float32, device=dev)
        self.outs = torch.zeros(rows, B, self.r, self.odim, dtype=torch.float32, device=dev)
        self.probs = torch.zeros(rows, B, self.r, dtype=torch.float32, device=dev)
        # the cross-attention record is opt-in: [rows, B, layers, H, S] fp32 is 3.6 GiB per 30 s utterance
        self.attn = torch.zeros(rows, B, L, H, self.S, dtype=torch.float32, device=dev) if attention else None
        self.stop = torch.zeros(rows, dtype=torch.int32, device=dev)  # every row done after step t
        self.done = torch.zeros(B, dtype=torch.bool, device=dev)
        self.lengths = torch.zeros(B, dtype=torch.int64, device=dev)
        self.minlen = torch.zeros(B, dtype=torch.int64, device=dev)
        self.maxlen_b = torch.zeros(B, dtype=torch.int64, device=dev)
        self.threshold = torch.full((1,), 0.5, dtype=torch.float32, device=dev)
        self.pos = torch.arange(rows, device=dev)
        pre = model.speech_decoder_prenet
        self.pe = pre.decoder_prenet[1].table(rows, dev)
        self.spk_bias = torch.zeros((B, pre.embed_dim), dtype=torch.float32, device=dev)
        self.with_spk = False
        self.graphs = {}
        self.stream = torch.cuda.Stream(device=dev) if capture else None
        self.dtype = RT.dtype
        # the graphs bake the address of the dropout seed they dereference and advance: it must be THIS object's tensor,
        # installed as the runtime's device seed for the duration of a synthesis (generate_speech restores the caller's)
        self.seed_t = torch.zeros(1, dtype=torch.int64, device=dev)

    @torch.no_grad()
    def begin(self, encoder_outs, spkembs, threshold, minlens, maxlens):
        """Load B utterances (one encoder output each, batch 1): project their cross-attention keys / values into rows
        of the static buffers, set their length limits, reset the counters. Returns their encoder lengths."""
        assert len(encoder_outs) == self.B and RT.dtype == self.dtype
        self.cache.enc_pad.fill_(1)
        lens = []
        for b, encoder_out in enumerate(encoder_outs):
            enc = encoder_out.get("_encoder_out_btc")
            if enc is None:
                enc = encoder_out["encoder_out"][0].transpose(0, 1).contiguous()
            enc = _act_dtype(enc)
            S = enc.shape[1]
            assert enc.shape[0] == 1 and S <= self.S
            pm = encoder_out["encoder_padding_mask"]
            self.cache.enc_pad[b, :S] = pm[0][0].to(torch.uint8) if len(pm) > 0 and pm[0] is not None else 0
            for li, layer in enumerate(self.m.decoder.layers):
                ca = layer.encoder_attn
                self.cache.cross[li][b:b + 1, :S] = ops.linear(enc, (ca.k_proj.weight, ca.v_proj.weight),
                                                               (ca.k_proj.bias, ca.v_proj.bias))
            lens.append(S)
        pre = self.m.speech_decoder_prenet
        with_spk = spkembs is not None
        if self.graphs and with_spk != self.with_spk:
            self.graphs = {}  # (the merge layer is part of the captured body)
        self.with_spk = with_spk
        if with_spk:  # (speech_decoder_prenet.py:76-89) the speaker half of the merge layer: once per utterance
            W, d = pre.spkembs_layer[0].weight, pre.embed_dim
            spk = torch.nn.functional.normalize(spkembs.float()).to(RT.dtype)
            self.spk_bias.copy_(ops.linear(spk, W[:, d:], (), out_dtype=torch.float32, key=("spk_w", id(W)), need_dx=False))
        self.threshold.fill_(float(threshold))
        self.minlen.copy_(torch.tensor(minlens, dtype=torch.int64))
        self.maxlen_b.copy_(torch.tensor(maxlens, dtype=torch.int64))
        self.done.zero_()
        self.lengths.zero_()
        self.t.zero_()
        self.ys_last.zero_()
        if self.capture:
            self.seed_t.fill_(RT._seed + (RT._draws << 20))  # a fresh stream of prenet masks per batch
            RT._draws += 1
            RT._seed_t = self.seed_t
        return lens

    def _body(self, span):
        m, pre, post = self.m, self.m.speech_decoder_prenet, self.m.speech_decoder_postnet
        taco, lin, pos = pre.decoder_prenet[0][0], pre.decoder_prenet[0][1], pre.decoder_prenet[1]
        x = self.ys_last.to(RT.dtype)
        for layer in taco.prenet:  # dropout in eval too (espnet Prenet semantics)
            x = ops.linear(x, layer[0].weight, layer[0].bias, act="relu", drop_p=taco.dropout_rate)
        x = ops.linear(x, lin.weight, lin.bias)
        x = ops.scaled_posenc(self.pe.index_select(0, self.t), pos.alpha, 0.0, x=x)
        if self.with_spk:
            W, b, d = pre.spkembs_layer[0].weight, pre.spkembs_layer[0].bias, pre.embed_dim
            x = ops.linear(x, W[:, :d], b, act="relu", bias2=self.spk_bias, bias2_rows=1, key=("spk_h", id(W)))
        self_pad = (self.pos[:span] > self.t).to(torch.uint8)[None].expand(self.B, span).contiguous()
        want = self.attn is not None
        z, layer_attn = decoder_step(m.decoder, x, self.cache, need_head_weights=want, t_dev=self.t, span=span,
                                     self_pad=self_pad)
        before, logits = post.project(z.contiguous())  # [B, r, odim], [B, r]
        p = torch.sigmoid(logits)
        self.outs.index_copy_(0, self.t, before[None])
        self.probs.index_copy_(0, self.t, p[None])
        if want:
            self.attn.index_copy_(0, self.t, torch.stack([a[:, :, 0, :] for a in layer_attn], 1)[None])
        self.ys_last.copy_(before[:, -1:, :])
        # (:1235-1245) per row: stop once a probability of the group reaches the threshold or idx >= maxlen, but not
        # before idx >= minlen; idx = t + 1 is the reference's counter after this step
        i = self.t + 1
        fin = ((p >= self.threshold).any(-1) | (i >= self.maxlen_b)) & (i >= self.minlen)
        newly = fin & ~self.done
        self.lengths.copy_(torch.where(newly, i.expand(self.B), self.lengths))
        self.done |= newly
        self.stop.index_copy_(0, self.t, self.done.all().to(torch.int32).reshape(1))
        self.t += 1
        RT.advance_seed()

    def _span(self, t):
        span = 128
        while span < t + 1:
            span *= 2
        return min(span, self.cache.max_len)

    def _snapshot(self):
        """State the step body overwrites that a replay of the same step does not rewrite first (capture warm-up)."""
        keep, done, lengths = self.ys_last.clone(), self.done.clone(), self.lengths.clone()

        def undo():
            self.seed_t -= 1  # (the pass drew from the seed the replay of this step must see)
            self.ys_last.copy_(keep)
            self.done.copy_(done)
            self.lengths.copy_(lengths)
        return undo

    @torch.no_grad()
    def run(self, t0, n):
        """Decoder steps t0 .. t0+n-1 (the device counter holds t0). Returns their stop flags (one device->host copy)."""
        for t in range(t0, t0 + n):
            span = self._span(t)
            if not self.capture:
                self._body(span)
                continue
            g = self.graphs.get(span)
            if g is None:
                # one eager pass builds every weight shadow and scratch outside the capture, then its effects are
                # undone: the cache row / result rows it wrote are rewritten by the replay of the same step
                self.stream.wait_stream(torch.cuda.current_stream(self.dev))
                with torch.cuda.stream(self.stream):
                    undo = self._snapshot()
                    self._body(span)
                    self.t -= 1
                    undo()
                    self.stream.synchronize()
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g, stream=self.stream):
                        self._body(span)
                torch.cuda.current_stream(self.dev).wait_stream(self.stream)
                self.graphs[span] = g
            g.replay()
        return self.stop[t0:t0 + n].tolist()

    @torch.no_grad()
    def synthesize(self, encoder_outs, spkembs, threshold, minlens, maxlens):
        """The reference's loop (:1222-1249) for every row: returns one (before frames [1, L_b, odim], stop
        probabilities [L_b], attention [layers, H, L_b/r, S_b] or None) per utterance."""
        assert max(maxlens) <= self.maxlen
        # (the reference's loop has no exit past maxlen frames otherwise)
        minlens = [min(mn, max(mx, 1)) for mn, mx in zip(minlens, maxlens)]
        S = self.begin(encoder_outs, spkembs, threshold, minlens, maxlens)
        last = max(max(mx, 1) for mx in maxlens)  # every row is done after this many steps
        idx = 0
        while True:
            n = max(1, min(self.CHUNK, last - idx))
            flags = self.run(idx, n)
            idx += n
            if any(flags):
                break
        res = []
        for b, L in enumerate(self.lengths.tolist()):
            attn = self.attn[:L, b, :, :, :S[b]].permute(1, 2, 0, 3).contiguous() if self.attn is not None else None
            res.append((self.outs[:L, b].reshape(1, L * self.r, self.odim).clone(), self.probs[:L, b].reshape(-1).clone(),
                        attn))
        return res


def synthesis_graph(model, S, maxlen, device, capture=True, B=1, attention=True):
    """The model's SynthesisGraph for B utterances, encoder length S and a frame budget of maxlen decoder steps
    (buckets: S to multiples of 64, maxlen to powers of two >= 256); rebuilt when the numeric mode or the weights'
    owner changed."""
    S_b = max(64, (S + 63) // 64 * 64)
    M_b = 256
    while M_b < maxlen:
        M_b *= 2
    store = model.__dict__.setdefault("_synthesis_graphs", {})
    key = (B, bool(attention), S_b, M_b, RT.dtype, str(device), bool(capture), RT.param_epoch)
    sg = store.get(key)
    if sg is None:
        for k in [k for k in store if k[:7] == key[:7]]:  # same buckets, stale weights
            del store[k]
        sg = store[key] = SynthesisGraph(model, S_b, M_b, device, capture=capture, B=B, attention=attention)
    return sg


class GreedyGraph:
    """Beam-1 text decoding (speecht5/sequence_generator.py:207-655 with ctc_weight 0 and no LM, as
    T5TransformerModel.generate_text_greedy states it) with every step = ONE CUDA-graph replay: embedding + position row
    of the newest token (gathered by the device step counter), the key/value-cached decoder, the vocabulary projection,
    log-softmax, the reference's score masking (:430-446) as one additive mask plus two step-dependent terms, arg-max,
    and the bookkeeping (token written at t+1, finished flags, lengths) -- all on the device. Utterance-independent like
    SynthesisGraph: encoder length and step budget are buckets, cross keys / values are copied into fixed buffers."""

    CHUNK = 8

    def __init__(self, model, B, S_bucket, maxlen_bucket, device, capture=True):
        self.m, self.capture = model, capture
        dec = model.decoder
        dev = torch.device(device)
        self.dev, self.B, self.S, self.maxlen = dev, int(B), int(S_bucket), int(maxlen_bucket)
        rows = self.maxlen + 1 + self.CHUNK
        C = dec.layers[0].self_attn.embed_dim
        self.cache = _StaticCache([torch.zeros((B, self.S, 2 * C), dtype=RT.dtype, device=dev) for _ in dec.layers],
                                  [torch.zeros((B, rows, 2 * C), dtype=RT.dtype, device=dev) for _ in dec.layers],
                                  torch.zeros((B, self.S), dtype=torch.uint8, device=dev), rows)
        self.t = torch.zeros(1, dtype=torch.int64, device=dev)
        self.tokens = torch.zeros((B, rows + 1), dtype=torch.long, device=dev)
        self.done = torch.zeros(B, dtype=torch.bool, device=dev)
        self.lengths = torch.zeros(B, dtype=torch.long, device=dev)
        self.stop = torch.zeros(rows, dtype=torch.int32, device=dev)
        self.pos_scores = torch.zeros((B, rows), dtype=torch.float32, device=dev)  # log-probability of the token emitted at t
        self.pos = torch.arange(rows, device=dev)
        pre = model.text_decoder_prenet
        self.pe = pre._table(rows, dev)
        V = model.text_decoder_postnet.output_projection.weight.shape[0]
        self.base_mask = torch.zeros(V, dtype=torch.float32, device=dev)   # pad / blank / mask symbol never, unk penalty
        self.only_eos = torch.zeros(V, dtype=torch.float32, device=dev)    # added once the step budget is reached
        self.eos_early = torch.zeros(V, dtype=torch.float32, device=dev)   # added while step < min_len
        self.min_len = torch.zeros(1, dtype=torch.int64, device=dev)
        self.max_len = torch.zeros(1, dtype=torch.int64, device=dev)
        self.inv_temp = torch.ones(1, dtype=torch.float32, device=dev)
        self.eos = 2
        self.graphs = {}
        self.stream = torch.cuda.Stream(device=dev) if capture else None
        self.dtype = RT.dtype

    @torch.no_grad()
    def begin(self, encoder_out, max_len, min_len, unk_penalty, temperature, pad, eos, unk, blank, mask_idx):
        import math
        enc = encoder_out.get("_encoder_out_btc")
        if enc is None:
            enc = encoder_out["encoder_out"][0].transpose(0, 1).contiguous()
        enc = _act_dtype(enc)
        B, S = enc.shape[0], enc.shape[1]
        assert B == self.B and S <= self.S and max_len <= self.maxlen and RT.dtype == self.dtype
        pm = encoder_out["encoder_padding_mask"]
        self.cache.enc_pad.fill_(1)
        self.cache.enc_pad[:, :S] = pm[0].to(torch.uint8) if len(pm) > 0 and pm[0] is not None else 0
        for li, layer in enumerate(self.m.decoder.layers):
            ca = layer.encoder_attn
            self.cache.cross[li][:, :S] = ops.linear(enc, (ca.k_proj.weight, ca.v_proj.weight),
                                                     (ca.k_proj.bias, ca.v_proj.bias))
        self.base_mask.zero_()
        self.base_mask[pad] = -math.inf
        self.base_mask[unk] -= unk_penalty
        self.base_mask[blank] = -math.inf
        if mask_idx is not None and mask_idx != unk:
            self.base_mask[mask_idx] = -math.inf
        self.only_eos.fill_(-math.inf)
        self.only_eos[eos] = 0.0
        self.eos_early.zero_()
        self.eos_early[eos] = -math.inf
        self.min_len.fill_(int(min_len))
        self.max_len.fill_(int(max_len))
        self.inv_temp.fill_(1.0 / float(temperature))
        if self.graphs and eos != self.eos:
            self.graphs = {}
        self.eos = int(eos)
        self.tokens.fill_(pad)
        self.tokens[:, 0] = eos
        self.done.zero_()
        self.lengths.zero_()
        self.t.zero_()

    def _body(self, span):
        m, pre = self.m, self.m.text_decoder_prenet
        tok = self.tokens.index_select(1, self.t).contiguous()  # [B, 1]
        x = ops.scaled_posenc(self.pe.index_select(0, self.t), pre._unit, 0.0, tokens=tok, emb=pre.embed_tokens.weight,
                              padding_idx=pre.padding_idx)
        self_pad = (self.pos[:span] > self.t).to(torch.uint8)[None].expand(self.B, span).contiguous()
        z, _ = decoder_step(m.decoder, x, self.cache, t_dev=self.t, span=span, self_pad=self_pad)
        logits = m.text_decoder_postnet(z)
        lp = torch.log_softmax(logits[:, -1, :].float() * self.inv_temp, dim=-1)
        lp = torch.where(lp != lp, torch.full_like(lp, float("-inf")), lp)
        zero = torch.zeros_like(self.base_mask)
        lp = lp + self.base_mask + torch.where(self.t < self.min_len, self.eos_early, zero) \
            + torch.where(self.t >= self.max_len, self.only_eos, zero)
        nxt = lp.argmax(dim=-1)
        self.tokens.index_copy_(1, self.t + 1, nxt[:, None])
        self.pos_scores.index_copy_(1, self.t, lp.gather(1, nxt[:, None]))
        newly = (~self.done) & nxt.eq(self.eos)
        self.lengths.copy_(torch.where(newly, (self.t + 1).expand(self.B), self.lengths))
        self.done |= newly
        self.stop.index_copy_(0, self.t, self.done.all().to(torch.int32).reshape(1))
        self.t += 1

    _span = SynthesisGraph._span
    run = SynthesisGraph.run

    def _snapshot(self):
        done, lengths = self.done.clone(), self.lengths.clone()

        def undo():  # (tokens[t+1] and stop[t] are rewritten by the replay; the finished flags are read-modify-write)
            self.done.copy_(done)
            self.lengths.copy_(lengths)
        return undo

    @torch.no_grad()
    def decode(self, encoder_out, max_len, **kw):
        """Returns a list of 1-D LongTensors ending in eos (generate_text_greedy's contract)."""
        self.begin(encoder_out, max_len, **kw)
        idx = 0
        while idx <= max_len:
            n = min(self.CHUNK, max_len + 1 - idx)
            flags = self.run(idx, n)
            idx += n
            if any(flags):
                break
        lengths = self.lengths.tolist()
        return [self.tokens[b, 1: lengths[b] + 1].clone() for b in range(self.B)]


def greedy_graph(model, B, S, max_len, device, capture=True):
    """The model's GreedyGraph for batch B, encoder length S and max_len steps (buckets: S to multiples of 64, max_len to
    powers of two >= 64); rebuilt when the numeric mode or the weights changed."""
    S_b = max(64, (S + 63) // 64 * 64)
    M_b = 64
    while M_b < max_len:
        M_b *= 2
    store = model.__dict__.setdefault("_greedy_graphs", {})
    key = (B, S_b, M_b, RT.dtype, str(device), bool(capture), RT.param_epoch)
    gg = store.get(key)
    if gg is None:
        for k in [k for k in store if k[:6] == key[:6]]:
            del store[k]
        gg = store[key] = GreedyGraph(model, B, S_b, M_b, device, capture=capture)
    return gg


class BeamGraph:
    """Beam search for text output (speecht5/sequence_generator.py:207-654 with ctc_weight 0, no LM, no prefix tokens;
    candidate selection fairseq/search.py:117-144) over B sentences x K beams = B*K decoder rows, every step = ONE
    CUDA-graph replay: embedding + position row of each row's newest token, the key/value-cached decoder, the vocabulary
    projection, st5_beam_topk (log-softmax, the reference's masking, the best min(2K, F-1) candidates per sentence) and
    st5_beam_update (finalize, is_finished, active selection, reorder) -- all on the device.

    The batch stays B*K rows: a finished sentence is skipped by the bookkeeping and what its rows still compute is never
    read (the reference drops it; every per-sentence quantity depends on that sentence only). A reorder never copies the
    key/value cache: each (row, position) cell is written once, and the lineage table lin[row][position] -- the
    self-attention's kv_rows -- says which row's cell holds each position of a hypothesis. Cross keys / values are
    projected once per sentence into [B, S, 2C]; the K beams read them with kv_div = K. Utterance-independent like
    GreedyGraph: encoder length and step budget are buckets. capture=False runs the same step body eagerly.

    With a language model `lm` (lm.TransformerLM, shallow fusion :420-426) the same replay also runs the LM one position
    per row -- embedding + position of the newest token, its layers on a [B*K, rows, 2C_lm] key/value cache per layer,
    its output projection -- and st5_beam_topk_lm adds lm_weight * log_softmax(LM logits) before the masking. The LM's
    cells are written once per (row, position) and read through the same lineage table, so a reorder moves no LM cache
    either. Token 0 of every hypothesis is eos for the LM as for the decoder."""

    CHUNK = 8

    def __init__(self, model, B, K, S_bucket, maxlen_bucket, device, capture=True, lm=None):
        self.m, self.capture = model, capture
        dec = model.decoder
        dev = torch.device(device)
        self.dev, self.B, self.K, self.S, self.maxlen = dev, int(B), int(K), int(S_bucket), int(maxlen_bucket)
        B, K = self.B, self.K
        BK = B * K
        rows = self.maxlen + 1 + self.CHUNK
        C = dec.layers[0].self_attn.embed_dim
        self.cache = _StaticCache([torch.zeros((B, self.S, 2 * C), dtype=RT.dtype, device=dev) for _ in dec.layers],
                                  [torch.zeros((BK, rows, 2 * C), dtype=RT.dtype, device=dev) for _ in dec.layers],
                                  torch.zeros((BK, self.S), dtype=torch.uint8, device=dev), rows)
        self.V = model.text_decoder_postnet.output_projection.weight.shape[0]
        i32, f32 = dict(dtype=torch.int32, device=dev), dict(dtype=torch.float32, device=dev)
        self.state = dict(
            t=torch.zeros(1, dtype=torch.int64, device=dev), max_len=torch.zeros(1, dtype=torch.int64, device=dev),
            cand_score=torch.zeros((B, 2 * K), **f32), cand_token=torch.zeros((B, 2 * K), **i32),
            cand_beam=torch.zeros((B, 2 * K), **i32), lin=torch.zeros((BK, rows), **i32),
            tok=torch.zeros((BK, rows), **i32), score=torch.zeros((BK, rows), **f32), ignore=torch.zeros(BK, **i32),
            finished=torch.zeros(B, **i32), parent=torch.zeros(BK, **i32),
            cur_tok=torch.zeros(BK, dtype=torch.int64, device=dev), cur_score=torch.zeros(BK, **f32),
            fin_n=torch.zeros(B, **i32), fin_tok=torch.zeros((B, K, rows), **i32),
            fin_pos=torch.zeros((B, K, rows), **f32), fin_len=torch.zeros((B, K), **i32),
            fin_score=torch.zeros((B, K), **f32), stop=torch.zeros(rows, **i32))
        self.t, self.stop = self.state["t"], self.state["stop"]
        self.min_len = torch.zeros(1, dtype=torch.int64, device=dev)
        self.mask = torch.zeros(self.V, dtype=torch.float32, device=dev)  # pad / blank / mask symbol never, unk penalty
        self.pos = torch.arange(rows, device=dev)
        self.pe = model.text_decoder_prenet._table(rows, dev)
        self.lm = lm
        if lm is not None:
            C_lm = lm.args.decoder_embed_dim
            self.lm_cache = _StaticCache([], [torch.zeros((BK, rows, 2 * C_lm), dtype=RT.dtype, device=dev)
                                              for _ in lm.decoder.layers], None, rows)
            self.lm_emb = torch.zeros((lm.vocab_size, C_lm), dtype=torch.float32, device=dev)  # embed_scale * E
            self.lm_pe = torch.zeros((rows, C_lm), dtype=torch.float32, device=dev)
        # (eos, 1 / temperature, normalize, len_penalty, lm_weight): host arguments the graphs bake
        self.consts = None
        self.graphs = {}
        self.stream = torch.cuda.Stream(device=dev) if capture else None
        self.dtype = RT.dtype

    @torch.no_grad()
    def begin(self, encoder_out, max_len, min_len, unk_penalty, temperature, pad, eos, unk, blank, mask_idx,
              normalize_scores, len_penalty, lm_weight=0.0):
        import math
        enc = encoder_out.get("_encoder_out_btc")
        if enc is None:
            enc = encoder_out["encoder_out"][0].transpose(0, 1).contiguous()
        enc = _act_dtype(enc)
        B, S = enc.shape[0], enc.shape[1]
        assert B == self.B and S <= self.S and max_len <= self.maxlen and RT.dtype == self.dtype
        pm = encoder_out["encoder_padding_mask"]
        self.cache.enc_pad.fill_(1)
        pad_rows = pm[0].to(torch.uint8) if len(pm) > 0 and pm[0] is not None else 0
        self.cache.enc_pad.view(B, self.K, self.S)[:, :, :S] = pad_rows[:, None] if torch.is_tensor(pad_rows) else 0
        for li, layer in enumerate(self.m.decoder.layers):
            ca = layer.encoder_attn
            self.cache.cross[li][:, :S] = ops.linear(enc, (ca.k_proj.weight, ca.v_proj.weight),
                                                     (ca.k_proj.bias, ca.v_proj.bias))
        self.mask.zero_()
        self.mask[pad] = -math.inf
        self.mask[unk] -= unk_penalty
        self.mask[blank] = -math.inf
        if mask_idx is not None and mask_idx != unk:
            self.mask[mask_idx] = -math.inf
        if self.lm is not None:  # (the tables the LM's graph body reads: refreshed for weights changed in place)
            self.lm_emb.copy_(self.lm.scaled_embedding())
            n = min(self.lm_pe.shape[0], max_len + 1)  # (positions past the step budget are never read)
            self.lm_pe.zero_()
            self.lm_pe[:n] = self.lm.positions(n, self.dev)
        consts = (int(eos), 1.0 / float(temperature), bool(normalize_scores), float(len_penalty), float(lm_weight))
        if self.graphs and consts != self.consts:
            self.graphs = {}
        self.consts = consts
        st = self.state
        self.min_len.fill_(int(min_len))
        st["max_len"].fill_(int(max_len))
        for n in ("lin", "tok", "score", "ignore", "finished", "parent", "cur_score", "fin_n", "stop", "t"):
            st[n].zero_()
        st["lin"][:, 0] = torch.arange(self.B * self.K, dtype=torch.int32, device=self.dev)
        st["cur_tok"].fill_(eos)

    def _body(self, span):
        m, pre, st = self.m, self.m.text_decoder_prenet, self.state
        eos, inv_temp, normalize, len_penalty, lm_weight = self.consts
        BK = self.B * self.K
        x = ops.scaled_posenc(self.pe.index_select(0, self.t), pre._unit, 0.0, tokens=st["cur_tok"].view(BK, 1),
                              emb=pre.embed_tokens.weight, padding_idx=pre.padding_idx)
        self_pad = (self.pos[:span] > self.t).to(torch.uint8)[None].expand(BK, span).contiguous()
        z, _ = decoder_step(m.decoder, x, self.cache, t_dev=self.t, span=span, self_pad=self_pad, self_rows=st["lin"],
                            cross_div=self.K)
        logits = m.text_decoder_postnet(z)
        fusion = {}  # (without an LM: st5_beam_topk)
        if self.lm is not None:
            y = ops.scaled_posenc(self.lm_pe.index_select(0, self.t), self.lm._unit, 0.0,
                                  tokens=st["cur_tok"].view(BK, 1), emb=self.lm_emb, padding_idx=self.lm.padding_idx)
            zl, _ = decoder_step(self.lm.decoder, y, self.lm_cache, t_dev=self.t, span=span, self_pad=self_pad,
                                 self_rows=st["lin"])
            fusion = dict(lm_logits=self.lm.output_layer(zl)[:, -1, :], lm_weight=lm_weight)
        kernels.beam_topk(logits[:, -1, :], st["cur_score"], self.mask, inv_temp, eos, self.t, self.min_len,
                          st["max_len"], st["cand_score"], st["cand_token"], st["cand_beam"], K=self.K, **fusion)
        kernels.beam_update(st, K=self.K, V=self.V, eos=eos, normalize=normalize, len_penalty=len_penalty)
        self.t += 1

    _span = SynthesisGraph._span
    run = SynthesisGraph.run

    def _snapshot(self):
        names = ("lin", "ignore", "finished", "cur_tok", "cur_score", "fin_n")
        keep = {n: self.state[n].clone() for n in names}

        def undo():  # (the lineage gather and the finalized counts are read-modify-write; the rest is rewritten)
            for n in names:
                self.state[n].copy_(keep[n])
        return undo

    @torch.no_grad()
    def decode(self, encoder_out, max_len, **kw):
        """Returns SequenceGenerator's hypotheses: per sentence, a list of its finalized hypotheses sorted by score
        descending (sequence_generator.py:644-654), each {"tokens", "score", "attention": None, "alignment",
        "positional_scores"}."""
        self.begin(encoder_out, max_len, **kw)
        idx = 0
        while idx <= max_len:
            n = min(self.CHUNK, max_len + 1 - idx)
            flags = self.run(idx, n)
            idx += n
            if any(flags):
                break
        st = self.state
        fin_n, fin_len = st["fin_n"].tolist(), st["fin_len"].tolist()
        fin_score, fin_tok, fin_pos = st["fin_score"].cpu(), st["fin_tok"].cpu(), st["fin_pos"].cpu()
        out = []
        for s in range(self.B):
            hyps = [{"tokens": fin_tok[s, i, :fin_len[s][i]].long().to(self.dev), "score": fin_score[s, i].to(self.dev),
                     "attention": None, "alignment": torch.empty(0),
                     "positional_scores": fin_pos[s, i, :fin_len[s][i]].to(self.dev)} for i in range(fin_n[s])]
            order = sorted(range(len(hyps)), key=lambda i: -float(fin_score[s, i]))
            out.append([hyps[i] for i in order])
        return out


def beam_graph(model, B, K, S, max_len, device, capture=True, lm=None):
    """The model's BeamGraph for B sentences x K beams, encoder length S and max_len steps (buckets: S to multiples of
    64, max_len to powers of two >= 64), fused with the language model `lm` or none; rebuilt when the numeric mode or
    the weights changed."""
    S_b = max(64, (S + 63) // 64 * 64)
    M_b = 64
    while M_b < max_len:
        M_b *= 2
    store = model.__dict__.setdefault("_beam_graphs", {})
    key = (B, K, S_b, M_b, RT.dtype, str(device), bool(capture), None if lm is None else id(lm), RT.param_epoch)
    bg = store.get(key)
    if bg is None:
        for k in [k for k in store if k[:8] == key[:8]]:
            del store[k]
        bg = store[key] = BeamGraph(model, B, K, S_b, M_b, device, capture=capture, lm=lm)
    return bg
