"""Shared Transformer encoder / decoder of SpeechT5 on the H100 kernel library.

Host-side mirror of the reference modules -- same class names, constructor arguments, parameter names and return
contracts -- with every tensor op routed to libspeecht5_b200.so through speecht5_b200.ops:
  MultiheadAttention              <- speecht5/models/modules/multihead_attention.py:23-522
  RelativePositionalEncoding      <- speecht5/models/modules/encoder.py:40-59
  TransformerSentenceEncoderLayer <- speecht5/models/modules/transformer_layer.py:23-134
  TransformerDecoderLayer         <- speecht5/models/modules/transformer_layer.py:137-411
  TransformerEncoder              <- speecht5/models/modules/encoder.py:61-380
  TransformerDecoder              <- speecht5/models/modules/decoder.py:33-324
Internally activations are batch-major [B, T, C] (token rows are the GEMM M dimension); module boundaries return the
reference layouts (encoder_out [T, B, C], attention weights [B, H, T, S])."""
import contextlib
import math

import numpy as np
import torch
import torch.nn as nn

from ... import ops
from ...ops import RT


def _act_dtype(x):
    return x if x.dtype == RT.dtype else x.to(RT.dtype)


def _fold_residual_grad(x):
    """Post-LN blocks: hand the block input to the residual add through the first GEMM's alias output, so that the
    residual branch's gradient is added in that GEMM's dx epilogue (only when a gradient will flow at all)."""
    return torch.is_grad_enabled() and x.requires_grad and ops.RT.fold_residual_grad


def _keep_or_skip(keep, y, x):
    """LayerDrop under CUDA-graph capture: the layer's output where `keep` (device 0/1 flag) is set, else its input --
    together with the fp32 copy of the residual stream (ops.residual_layer_norm), so that the next layer adds the same
    residual an eager update that ran or skipped this layer would. A side without a copy (the stack's input) is a bf16
    tensor whose fp32 value is exact."""
    on = keep > 0.5
    out = torch.where(on, y, x)
    y32, x32 = getattr(y, "_st5_f32", None), getattr(x, "_st5_f32", None)
    if y32 is not None or x32 is not None:
        out._st5_f32 = torch.where(on, y32 if y32 is not None else y.float(), x32 if x32 is not None else x.float())
    return out


class MultiheadAttention(nn.Module):
    """Parameter holder with the reference's names (q/k/v/out_proj Linear); compute happens in the owning layer through
    ops.linear (fused q|k|v projection) + ops.attention."""

    def __init__(self, embed_dim, num_heads, kdim=None, vdim=None, dropout=0.0, bias=True, self_attention=False,
                 encoder_decoder_attention=False, has_relative_attention_bias=False, head_dims=(64,)):
        super().__init__()
        self.embed_dim = embed_dim
        self.kdim = kdim if kdim is not None else embed_dim
        self.vdim = vdim if vdim is not None else embed_dim
        self.num_heads = num_heads
        self.dropout_p = dropout
        self.head_dim = embed_dim // num_heads
        assert self.head_dim * num_heads == embed_dim, "embed_dim must be divisible by num_heads"
        # head_dims: the widths this module may be built with. The speech model's attention (fused kernels, training) takes
        # 64; the fusion LM (lm.TransformerLM, evaluation only) also 80, on the one-row kernel (ops.attention_rows).
        assert self.head_dim in head_dims, f"head_dim {self.head_dim}: the attention kernels here take {head_dims}"
        self.scaling = self.head_dim ** -0.5
        self.self_attention = self_attention
        self.encoder_decoder_attention = encoder_decoder_attention
        self.has_relative_attention_bias = has_relative_attention_bias
        self.k_proj = nn.Linear(self.kdim, embed_dim, bias=bias)
        self.v_proj = nn.Linear(self.vdim, embed_dim, bias=bias)
        self.q_proj = nn.Linear(embed_dim, embed_dim, bias=bias)
        self.out_proj = nn.Linear(embed_dim, embed_dim, bias=bias)
        self.reset_parameters()

    def reset_parameters(self):  # multihead_attention.py:100-118
        g = 1 / math.sqrt(2)
        nn.init.xavier_uniform_(self.k_proj.weight, gain=g)
        nn.init.xavier_uniform_(self.v_proj.weight, gain=g)
        nn.init.xavier_uniform_(self.q_proj.weight, gain=g)
        nn.init.xavier_uniform_(self.out_proj.weight)
        if self.out_proj.bias is not None:
            nn.init.constant_(self.out_proj.bias, 0.0)

    def self_attend(self, x, key_padding_mask=None, causal=False, pe_k=None, maxpos=0, training=True, passthrough=False):
        """x [B,T,C] -> attention output before out_proj, [B,T,C]. passthrough: also return the alias of x the caller
        must use for its residual add (ops.LinearFn: the residual branch's gradient is then added in the dx GEMM)."""
        x_pt = None
        if passthrough:
            qkv, x_pt = ops.linear(x, (self.q_proj.weight, self.k_proj.weight, self.v_proj.weight),
                                   (self.q_proj.bias, self.k_proj.bias, self.v_proj.bias), passthrough=True)
        else:
            qkv = ops.linear(x, (self.q_proj.weight, self.k_proj.weight, self.v_proj.weight),
                             (self.q_proj.bias, self.k_proj.bias, self.v_proj.bias))
        out, _ = ops.attention(qkv, None, H=self.num_heads, d=self.embed_dim, q_col=0, k_col=1, v_col=2,
                               scale=self.scaling, pe_k=pe_k if self.has_relative_attention_bias else None,
                               maxpos=maxpos, key_pad=key_padding_mask, causal=causal,
                               drop_p=self.dropout_p if training else 0.0)
        return (out, x_pt) if passthrough else out

    def cross_attend(self, x, enc, key_padding_mask=None, need_head_weights=False, training=True, passthrough=False):
        """x [B,Tq,C], enc [B,Tk,C] -> (attention output before out_proj, probs [B,H,Tq,Tk] fp32 or None[, alias of x])."""
        x_pt = None
        if passthrough:
            q, x_pt = ops.linear(x, self.q_proj.weight, self.q_proj.bias, passthrough=True)
        else:
            q = ops.linear(x, self.q_proj.weight, self.q_proj.bias)
        kv = ops.linear(enc, (self.k_proj.weight, self.v_proj.weight), (self.k_proj.bias, self.v_proj.bias))
        out, probs = ops.attention(q, kv, H=self.num_heads, d=self.embed_dim, q_col=0, k_col=0, v_col=1,
                                   scale=self.scaling, key_pad=key_padding_mask,
                                   drop_p=self.dropout_p if training else 0.0, return_probs=need_head_weights)
        if passthrough:
            return out, (probs if need_head_weights else None), x_pt
        return out, (probs if need_head_weights else None)


class RelativePositionalEncoding(nn.Module):
    """Table holder (pe_k [2*maxlen, d_head]); the T x T x 64 gather of the reference is never materialised -- the
    attention kernel indexes the table with clamp(i - j)."""

    def __init__(self, d_model, maxlen=1000, embed_v=False):
        super().__init__()
        self.d_model, self.maxlen, self.embed_v = d_model, maxlen, embed_v
        self.pe_k = nn.Embedding(2 * maxlen, d_model)
        if embed_v:
            self.pe_v = nn.Embedding(2 * maxlen, d_model)


class TransformerSentenceEncoderLayer(nn.Module):
    def __init__(self, embedding_dim=768, ffn_embedding_dim=3072, num_attention_heads=8, dropout=0.1,
                 attention_dropout=0.1, activation_dropout=0.1, activation_fn="relu", layer_norm_first=False,
                 has_relative_attention_bias=False):
        super().__init__()
        self.embedding_dim, self.dropout, self.activation_dropout = embedding_dim, dropout, activation_dropout
        assert activation_fn in ("gelu", "relu")
        self.activation_fn = activation_fn
        self.self_attn = MultiheadAttention(embedding_dim, num_attention_heads, dropout=attention_dropout,
                                            self_attention=True, has_relative_attention_bias=has_relative_attention_bias)
        self.layer_norm_first = layer_norm_first
        self.self_attn_layer_norm = nn.LayerNorm(embedding_dim)
        self.fc1 = nn.Linear(embedding_dim, ffn_embedding_dim)
        self.fc2 = nn.Linear(ffn_embedding_dim, embedding_dim)
        self.final_layer_norm = nn.LayerNorm(embedding_dim)
        if has_relative_attention_bias:
            self.norm_k = nn.LayerNorm(embedding_dim // num_attention_heads)

    def forward(self, x, self_attn_padding_mask=None, pos_bias=None, maxpos=0):
        """x [B,T,C]; pos_bias = the [2*maxpos, 64] table (fp32)."""
        tr = self.training
        p, pa = (self.dropout if tr else 0.0), (self.activation_dropout if tr else 0.0)
        if self.layer_norm_first:  # transformer_layer.py:90-111
            residual = x
            h = ops.residual_layer_norm(x, None, self.self_attn_layer_norm)
            if pos_bias is not None:
                pos_bias = ops.residual_layer_norm(pos_bias, None, self.norm_k)
            a = self.self_attn.self_attend(h, self_attn_padding_mask, pe_k=pos_bias, maxpos=maxpos, training=tr)
            x = ops.linear(a, self.self_attn.out_proj.weight, self.self_attn.out_proj.bias, drop_p=p, residual=residual)
            residual = x
            h = ops.residual_layer_norm(x, None, self.final_layer_norm)
            x = ops.ffn(h, self.fc1, self.fc2, self.activation_fn, drop_a=pa, drop_o=p, residual=residual)
        else:  # :112-132
            # (the block input reaches the residual add as the alias its first GEMM hands back: ops.LinearFn.forward)
            pt = _fold_residual_grad(x)
            a = self.self_attn.self_attend(x, self_attn_padding_mask, pe_k=pos_bias, maxpos=maxpos, training=tr, passthrough=pt)
            a, r = a if pt else (a, x)
            o = ops.linear(a, self.self_attn.out_proj.weight, self.self_attn.out_proj.bias, bias_grad_by_consumer=True)
            x = ops.residual_layer_norm(o, r, self.self_attn_layer_norm, drop_p=p, stream=True)
            pt = _fold_residual_grad(x)
            o = ops.ffn(x, self.fc1, self.fc2, self.activation_fn, drop_a=pa, passthrough=pt, bias_grad_by_consumer=True)
            o, r = o if pt else (o, x)
            x = ops.residual_layer_norm(o, r, self.final_layer_norm, drop_p=p, stream=True)
        return x, None


class TransformerEncoder(nn.Module):
    def __init__(self, args, tgt_dict=None, embed_tokens=None):
        super().__init__()
        self.args = args
        self.register_buffer("version", torch.Tensor([3]))
        self.dropout_p = args.dropout
        self.encoder_layerdrop = args.encoder_layerdrop
        self.freeze_encoder_updates = args.freeze_encoder_updates
        self.no_freeze_encoder_layer = (eval(args.no_freeze_encoder_layer)
                                        if getattr(args, "no_freeze_encoder_layer", None) is not None else None)
        self.num_updates = 0
        assert getattr(args, "use_sent_enc_layer", True), "only the SentenceEncoderLayer encoder is implemented"
        self.layers = nn.ModuleList([self.build_encoder_layer(args) for _ in range(args.encoder_layers)])
        self.num_layers = len(self.layers)
        self.use_sent_enc_layer = True
        self.unb_enc_layer = getattr(args, "unb_enc_layer", -1)
        self.layer_norm_first = args.layer_norm_first
        self.layer_norm = nn.LayerNorm(args.encoder_embed_dim, eps=args.layer_norm_eps)
        if args.share_ctc_embed and embed_tokens is not None:
            self.proj = nn.Linear(embed_tokens.weight.shape[1], embed_tokens.weight.shape[0], bias=False)
            self.proj.weight = embed_tokens.weight
        elif tgt_dict is not None:
            self.proj = nn.Linear(args.encoder_embed_dim, len(tgt_dict))
            nn.init.xavier_uniform_(self.proj.weight)
            nn.init.constant_(self.proj.bias, 0.0)
        else:
            self.proj = None
        if args.relative_position_embedding:
            self.pos_emb = RelativePositionalEncoding(args.encoder_embed_dim // args.encoder_attention_heads,
                                                      args.encoder_max_relative_position)

    def build_encoder_layer(self, args):
        return TransformerSentenceEncoderLayer(
            embedding_dim=args.encoder_embed_dim, ffn_embedding_dim=args.encoder_ffn_embed_dim,
            num_attention_heads=args.encoder_attention_heads, dropout=args.dropout,
            attention_dropout=args.attention_dropout, activation_dropout=args.activation_dropout,
            activation_fn=args.activation_fn, layer_norm_first=args.layer_norm_first,
            has_relative_attention_bias=args.relative_position_embedding)

    def forward(self, encoder_in, encoder_padding_mask, return_all_hiddens=False, tgt_layer=None):
        ft = self.freeze_encoder_updates <= self.num_updates if self.no_freeze_encoder_layer is None else True
        with torch.no_grad() if not ft else contextlib.ExitStack():
            encoder_out = self.forward_scriptable(encoder_in, encoder_padding_mask, return_all_hiddens, tgt_layer)
        if self.proj is not None:  # encoder.py:173-179 CTC head on dropout(x)
            x_tbc = encoder_out["encoder_out"][0]
            xb = ops.dropout(encoder_out["_encoder_out_btc"], self.dropout_p, self.training)
            ctc = ops.linear(xb, self.proj.weight, self.proj.bias, out_dtype=torch.float32).transpose(0, 1)
            assert ctc.shape[0] == x_tbc.shape[0]
            encoder_out["encoder_out_for_ctc"] = [ctc]
        else:
            encoder_out["encoder_out_for_ctc"] = [None]
        return encoder_out

    def forward_scriptable(self, encoder_in, encoder_padding_mask, return_all_hiddens=False, tgt_layer=None):
        ft = self.freeze_encoder_updates <= self.num_updates if self.no_freeze_encoder_layer is not None else True
        with torch.no_grad() if not ft else contextlib.ExitStack():
            x = _act_dtype(encoder_in)
            if not self.layer_norm_first:
                x = ops.residual_layer_norm(x, None, self.layer_norm, stream=True)
            x = ops.dropout(x, self.dropout_p, self.training)
            encoder_states = []
            if return_all_hiddens:
                encoder_states.append(x.transpose(0, 1))
            pos_k, maxpos = None, 0
            if self.args.relative_position_embedding:
                pos_k, maxpos = self.pos_emb.pe_k.weight, self.pos_emb.maxlen
        r = d = None
        keep_dev, keep_host = RT.layer_keep, RT.layer_keep_host
        blocks, base = self.training and (keep_dev is not None or keep_host is not None), RT._offset
        for i, layer in enumerate(self.layers):
            x = RT.stage(("enc", i), x)  # gradient-exchange overlap point (trainer), identity otherwise
            if blocks:
                RT.offset_block(base, i)
            frozen = (not ft) and i not in self.no_freeze_encoder_layer
            with torch.no_grad() if frozen else contextlib.ExitStack():
                if self.training and keep_dev is not None:
                    # LayerDrop under CUDA-graph capture: the trainer drew the subset (same numpy stream as :252); a
                    # dropped layer's output is replaced by its input, its parameters receive exactly zero gradient
                    y, _ = layer(x, self_attn_padding_mask=encoder_padding_mask, pos_bias=pos_k, maxpos=maxpos)
                    x = _keep_or_skip(keep_dev[i], y, x)
                else:
                    if keep_host is not None:
                        run = bool(keep_host[i] > 0.5)
                    else:
                        dropout_probability = np.random.random()  # numpy RNG, as encoder.py:252
                        run = (dropout_probability > self.encoder_layerdrop) or i == self.unb_enc_layer
                    if not self.training or run:
                        x, _ = layer(x, self_attn_padding_mask=encoder_padding_mask, pos_bias=pos_k, maxpos=maxpos)
                if i == self.unb_enc_layer:
                    d = x
                if i == tgt_layer:
                    r = x
                    break
                if return_all_hiddens:
                    encoder_states.append(x.transpose(0, 1))
        if blocks:
            RT.offset_block(base, len(self.layers))
        with torch.no_grad() if not ft else contextlib.ExitStack():
            if self.layer_norm_first:
                x = ops.residual_layer_norm(x, None, self.layer_norm)
            if r is not None:
                x = r
        return {
            "encoder_out": [x.transpose(0, 1)],  # T x B x C (reference layout)
            "_encoder_out_btc": x,                # B x T x C (kernel layout, consumed by our decoder)
            "encoder_padding_mask": [encoder_padding_mask],
            "encoder_states": encoder_states,
            "src_tokens": [],
            "decoder_input": [d.transpose(0, 1) if d is not None else None],
        }

    def reorder_encoder_out(self, encoder_out, new_order):  # encoder.py:293-333
        new = dict(encoder_out)
        if len(encoder_out["encoder_out"]) > 0:
            new["encoder_out"] = [encoder_out["encoder_out"][0].index_select(1, new_order)]
            new["_encoder_out_btc"] = encoder_out["_encoder_out_btc"].index_select(0, new_order)
        if len(encoder_out["encoder_padding_mask"]) > 0 and encoder_out["encoder_padding_mask"][0] is not None:
            new["encoder_padding_mask"] = [encoder_out["encoder_padding_mask"][0].index_select(0, new_order)]
        if len(encoder_out.get("encoder_out_for_ctc", [])) > 0 and encoder_out["encoder_out_for_ctc"][0] is not None:
            new["encoder_out_for_ctc"] = [encoder_out["encoder_out_for_ctc"][0].index_select(1, new_order)]
        return new

    def set_num_updates(self, num_updates):
        self.num_updates = num_updates


class TransformerDecoderLayer(nn.Module):
    def __init__(self, args, no_encoder_attn=False, has_relative_attention_bias=False, head_dims=(64,)):
        super().__init__()
        self.embed_dim = args.decoder_embed_dim
        self.num_updates = 0
        self.dropout_p = args.dropout
        self.freeze_decoder_updates = getattr(args, "freeze_decoder_updates", 0)
        # decoder self-attention has NO relative bias in the reference (transformer_layer.py:229-242, kwarg commented
        # out at :241): the position table and norm_k below are dead parameters kept for checkpoint compatibility.
        self.self_attn = MultiheadAttention(self.embed_dim, args.decoder_attention_heads,
                                            dropout=args.attention_dropout, self_attention=True, head_dims=head_dims)
        act = getattr(args, "activation_fn", None) or "relu"
        assert act in ("gelu", "relu")
        self.activation_fn = act
        self.activation_dropout_p = float(getattr(args, "activation_dropout", 0) or getattr(args, "relu_dropout", 0) or 0)
        self.normalize_before = args.decoder_normalize_before
        self.self_attn_layer_norm = nn.LayerNorm(self.embed_dim)
        if no_encoder_attn:
            self.encoder_attn = self.encoder_attn_layer_norm = None
        else:
            self.encoder_attn = MultiheadAttention(self.embed_dim, args.decoder_attention_heads,
                                                   kdim=getattr(args, "encoder_embed_dim", None),
                                                   vdim=getattr(args, "encoder_embed_dim", None),
                                                   dropout=args.attention_dropout, encoder_decoder_attention=True)
            self.encoder_attn_layer_norm = nn.LayerNorm(self.embed_dim)
        self.fc1 = nn.Linear(self.embed_dim, args.decoder_ffn_embed_dim)
        self.fc2 = nn.Linear(args.decoder_ffn_embed_dim, self.embed_dim)
        self.final_layer_norm = nn.LayerNorm(self.embed_dim)
        self.need_attn = True
        self.has_relative_attention_bias = has_relative_attention_bias
        if has_relative_attention_bias:
            self.norm_k = nn.LayerNorm(self.embed_dim // args.decoder_attention_heads)

    def forward(self, x, encoder_out=None, encoder_padding_mask=None, causal=True, self_attn_padding_mask=None,
                need_attn=False, need_head_weights=False):
        """x [B,T,C], encoder_out [B,S,C] -> (x, attn [B,H,T,S] fp32 or None)."""
        ft = self.freeze_decoder_updates <= self.num_updates
        tr = self.training
        p, pa = (self.dropout_p if tr else 0.0), (self.activation_dropout_p if tr else 0.0)
        if need_head_weights:
            need_attn = True
        with torch.no_grad() if not ft else contextlib.ExitStack():
            if self.normalize_before:
                residual = x
                h = ops.residual_layer_norm(x, None, self.self_attn_layer_norm)
                a = self.self_attn.self_attend(h, self_attn_padding_mask, causal=causal, training=tr)
                x = ops.linear(a, self.self_attn.out_proj.weight, self.self_attn.out_proj.bias, drop_p=p,
                               residual=residual)
            else:
                pt = _fold_residual_grad(x)
                a = self.self_attn.self_attend(x, self_attn_padding_mask, causal=causal, training=tr, passthrough=pt)
                a, r = a if pt else (a, x)
                o = ops.linear(a, self.self_attn.out_proj.weight, self.self_attn.out_proj.bias,
                               bias_grad_by_consumer=True)
                x = ops.residual_layer_norm(o, r, self.self_attn_layer_norm, drop_p=p, stream=True)
        attn = None
        if self.encoder_attn is not None and encoder_out is not None:
            want = need_attn or (not self.training and self.need_attn)
            if self.normalize_before:
                residual = x
                h = ops.residual_layer_norm(x, None, self.encoder_attn_layer_norm)
                a, attn = self.encoder_attn.cross_attend(h, encoder_out, encoder_padding_mask, want, tr)
                x = ops.linear(a, self.encoder_attn.out_proj.weight, self.encoder_attn.out_proj.bias, drop_p=p,
                               residual=residual)
            else:
                pt = _fold_residual_grad(x)
                res = self.encoder_attn.cross_attend(x, encoder_out, encoder_padding_mask, want, tr, passthrough=pt)
                a, attn, r = res if pt else (res[0], res[1], x)
                o = ops.linear(a, self.encoder_attn.out_proj.weight, self.encoder_attn.out_proj.bias,
                               bias_grad_by_consumer=True)
                x = ops.residual_layer_norm(o, r, self.encoder_attn_layer_norm, drop_p=p, stream=True)
            if attn is not None and not need_head_weights:
                attn = attn.mean(dim=1)
        with torch.no_grad() if not ft else contextlib.ExitStack():
            if self.normalize_before:
                residual = x
                h = ops.residual_layer_norm(x, None, self.final_layer_norm)
                x = ops.ffn(h, self.fc1, self.fc2, self.activation_fn, drop_a=pa, drop_o=p, residual=residual)
            else:
                pt = _fold_residual_grad(x)
                o = ops.ffn(x, self.fc1, self.fc2, self.activation_fn, drop_a=pa, passthrough=pt,
                            bias_grad_by_consumer=True)
                o, r = o if pt else (o, x)
                x = ops.residual_layer_norm(o, r, self.final_layer_norm, drop_p=p, stream=True)
        return x, attn, None

    def set_num_updates(self, num_updates):
        self.num_updates = num_updates


class TransformerDecoder(nn.Module):
    def __init__(self, args, no_encoder_attn=False):
        super().__init__()
        self.args = args
        self.register_buffer("version", torch.Tensor([3]))
        self.dropout_p = args.dropout
        self.decoder_layerdrop = args.decoder_layerdrop
        self.layers = nn.ModuleList([
            TransformerDecoderLayer(args, no_encoder_attn, has_relative_attention_bias=args.relative_position_embedding)
            for _ in range(args.decoder_layers)])
        self.num_layers = len(self.layers)
        if args.decoder_normalize_before and not getattr(args, "no_decoder_final_norm", False):
            self.layer_norm = nn.LayerNorm(args.decoder_embed_dim, eps=args.layer_norm_eps)
        else:
            self.layer_norm = None
        if args.relative_position_embedding:  # dead table, see TransformerDecoderLayer (decoder.py:83-84)
            self.pos_emb = RelativePositionalEncoding(args.encoder_embed_dim // args.encoder_attention_heads,
                                                      args.decoder_max_relative_position)

    def forward(self, prev_output_tokens, tgt_mask, encoder_out=None, incremental_state=None,
                full_context_alignment=False, alignment_layer=None, alignment_heads=None, src_lengths=None,
                return_all_hiddens=False):
        if incremental_state is not None:
            raise NotImplementedError("fairseq's incremental_state protocol is not used here: the key/value cache and "
                                      "the per-step CUDA graphs live in speecht5_b200/incremental.py")
        return self.extract_features(prev_output_tokens, tgt_mask, encoder_out, full_context_alignment,
                                     alignment_layer, alignment_heads)

    def extract_features(self, prev_output_tokens, tgt_mask, encoder_out, full_context_alignment=False,
                         alignment_layer=None, alignment_heads=None):
        """prev_output_tokens: decoder-prenet output [B,T,C]. Returns (x [B,T,C], {"attn": [...], ...})."""
        if alignment_layer is None:
            alignment_layer = self.num_layers - 1
        enc = padding_mask = None
        if encoder_out is not None and len(encoder_out["encoder_out"]) > 0:
            enc = encoder_out.get("_encoder_out_btc")
            if enc is None:
                enc = encoder_out["encoder_out"][0].transpose(0, 1).contiguous()
            enc = _act_dtype(enc)
        if encoder_out is not None and len(encoder_out["encoder_padding_mask"]) > 0:
            padding_mask = encoder_out["encoder_padding_mask"][0]
        x = _act_dtype(prev_output_tokens)
        attn_list, attn = [], None
        inner_states = [x]
        keep_dev, keep_host = RT.layer_keep, RT.layer_keep_host
        n_enc = 0 if (keep_dev is None and keep_host is None) else (len(keep_dev if keep_dev is not None else keep_host)
                                                                    - len(self.layers))
        blocks, base = self.training and (keep_dev is not None or keep_host is not None), RT._offset
        for idx, layer in enumerate(self.layers):
            x = RT.stage(("dec", idx), x)  # gradient-exchange overlap point (trainer), identity otherwise
            if blocks:
                RT.offset_block(base, idx)
            want = bool(idx == alignment_layer or alignment_layer == -1)
            if self.training and keep_dev is not None:  # LayerDrop under capture: see TransformerEncoder
                y, layer_attn, _ = layer(x, enc, padding_mask, causal=not full_context_alignment,
                                         self_attn_padding_mask=tgt_mask, need_attn=want, need_head_weights=want)
                x = _keep_or_skip(keep_dev[n_enc + idx], y, x)
                # (the reference drops the layer's attention map from the list too; under a static graph it stays, the
                #  s2t / pre-training criteria that use LayerDrop do not read it)
            else:
                if self.training and keep_host is not None:
                    if not bool(keep_host[n_enc + idx] > 0.5):
                        continue
                elif self.training and self.decoder_layerdrop > 0:  # fairseq LayerDropModuleList (torch RNG)
                    if torch.empty(1).uniform_().item() <= self.decoder_layerdrop:
                        continue
                x, layer_attn, _ = layer(x, enc, padding_mask, causal=not full_context_alignment,
                                         self_attn_padding_mask=tgt_mask, need_attn=want, need_head_weights=want)
            inner_states.append(x)
            if layer_attn is not None and want:
                attn = layer_attn.float()
                attn_list.append(attn)  # [B,H,T,S] == reference attn.transpose(0, 1)
        if blocks:
            RT.offset_block(base, len(self.layers))
        if attn is not None and len(attn_list) == 1:
            if alignment_heads is not None:
                attn = attn[:, :alignment_heads]
            attn = attn.mean(dim=1)
        if self.layer_norm is not None:
            x = ops.residual_layer_norm(x, None, self.layer_norm)
        return x, {"attn": [attn if len(attn_list) <= 1 else attn_list], "inner_states": inner_states}

    def set_num_updates(self, num_updates):
        for layer in self.layers:
            layer.set_num_updates(num_updates)
