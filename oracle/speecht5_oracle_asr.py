"""CPU restatement (oracle) of the speech-in / text-out (s2t, ASR fine-tune) path of microsoft/SpeechT5 -- SURVEY.md
section 8a rows 2, 3, 9, 14, 18, the "next" rows after the TTS step. TEST INFRASTRUCTURE ONLY: nothing in the product
path may import this file (only tests/, __graft_entry__.smoke() and bench.py's CPU legs may).

Every class cites the reference file:line it restates (paths under /root/reference/SpeechT5/speecht5 or
/root/reference/SpeechT5/fairseq/fairseq). The encoder / decoder stacks are the ones of oracle/speecht5_oracle.py.
Pinned against the independent HuggingFace port (transformers SpeechT5ForSpeechToText) by oracle/hf_crosscheck_asr.py;
the reference itself ships no golden vector for this path ("parity unpinned by the reference's own tests")."""
import math

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .speecht5_oracle import TransformerDecoder, TransformerEncoder, base_args, init_bert_params

CONV_FEATURE_LAYERS = [(512, 10, 5)] + [(512, 3, 2)] * 4 + [(512, 2, 2)] * 2  # models/speecht5.py:1345


def base_asr_args(**overrides):
    """t5_transformer_base_asr (models/speecht5.py:1427-1446) on top of base_architecture; LayerDrop / masking are
    host-RNG driven in the reference (numpy), so the deterministic oracle defaults them off -- pass them to enable."""
    kw = dict(activation_dropout=0.1, attention_dropout=0.1, dropout=0.1, feature_grad_mult=0.0, encoder_layerdrop=0.0,
              decoder_layerdrop=0.0, mask_prob=0.0, mask_channel_prob=0.0, hubert_mask_length=10,
              mask_channel_length=64, max_text_positions=600, max_speech_positions=4000, use_conv_pos=True,
              use_sinc_pos=True, conv_pos=128, conv_pos_groups=16, extractor_mode="default", conv_bias=False,
              no_scale_embedding=True, share_input_output_embed=False, share_ctc_embed=False,
              decoder_learned_pos=False, no_token_positional_embeddings=False, layernorm_embedding=False,
              conv_feature_layers=CONV_FEATURE_LAYERS)
    kw.update(overrides)
    return base_args(**kw)


# ------------------------------------------------------------------------------------------------ positions
def make_positions(tokens, padding_idx):
    """fairseq/utils.py:247-257: non-pad symbols are numbered from padding_idx + 1, pads keep padding_idx."""
    mask = tokens.ne(padding_idx).int()
    return (torch.cumsum(mask, dim=1).type_as(mask) * mask).long() + padding_idx


def sinusoidal_table(num_embeddings, dim, padding_idx):
    """fairseq/modules/sinusoidal_positional_embedding.py:36-58: [sin | cos] halves (tensor2tensor layout), divisor
    half_dim - 1, zero row at padding_idx."""
    half = dim // 2
    step = math.log(10000) / (half - 1)
    freq = torch.exp(torch.arange(half, dtype=torch.float) * -step)
    ang = torch.arange(num_embeddings, dtype=torch.float)[:, None] * freq[None, :]
    emb = torch.cat([torch.sin(ang), torch.cos(ang)], dim=1).view(num_embeddings, -1)
    if dim % 2 == 1:
        emb = torch.cat([emb, torch.zeros(num_embeddings, 1)], dim=1)
    emb[padding_idx, :] = 0
    return emb


class SinusoidalPositionalEmbedding(nn.Module):
    """fairseq/modules/sinusoidal_positional_embedding.py:60-105 without incremental state. `tokens` may be a boolean
    padding mask (speech prenet, speech_encoder_prenet.py:196-198): False != padding_idx(1) counts as a symbol."""

    def __init__(self, dim, padding_idx):
        super().__init__()
        self.dim, self.padding_idx = dim, padding_idx

    def forward(self, tokens):
        B, T = tokens.shape
        table = sinusoidal_table(self.padding_idx + 1 + T, self.dim, self.padding_idx)
        pos = make_positions(tokens, self.padding_idx)
        return table.index_select(0, pos.view(-1)).view(B, T, -1)


# ------------------------------------------------------------------------------------------------ speech encoder prenet
class ConvFeatureExtractionModel(nn.Module):
    """modules/speech_encoder_prenet.py:277-374. mode "default": GroupNorm(dim groups) after the first conv only;
    "layer_norm": LayerNorm over channels after every conv. Convs have no bias (conv_bias False), kaiming-normal."""

    def __init__(self, conv_layers=CONV_FEATURE_LAYERS, mode="default", conv_bias=False):
        super().__init__()
        assert mode in ("default", "layer_norm")
        self.mode = mode
        self.specs = list(conv_layers)
        self.conv_layers = nn.ModuleList()
        in_d = 1
        for i, (dim, k, stride) in enumerate(self.specs):
            conv = nn.Conv1d(in_d, dim, k, stride=stride, bias=conv_bias)
            nn.init.kaiming_normal_(conv.weight)
            mods = [conv, nn.Dropout(0.0)]
            if mode == "layer_norm":
                mods.append(nn.LayerNorm(dim))  # applied on the transposed tensor in forward()
            elif i == 0:
                mods.append(nn.GroupNorm(dim, dim, affine=True))
            mods.append(nn.GELU())
            self.conv_layers.append(nn.Sequential(*mods))
            in_d = dim

    def forward(self, x):  # [B, N] -> [B, C, T]
        x = x.unsqueeze(1)
        for blk in self.conv_layers:
            for m in blk:
                # Fp32LayerNorm (between TransposeLast) / Fp32GroupNorm: input AND affine parameters in (at least) fp32
                hi = x if x.dtype in (torch.float32, torch.float64) else x.float()
                w, b = (None if v is None else v.to(hi.dtype)
                        for v in (getattr(m, "weight", None), getattr(m, "bias", None)))
                if isinstance(m, nn.LayerNorm):
                    x = F.layer_norm(hi.transpose(1, 2), m.normalized_shape, w, b, m.eps).transpose(1, 2).type_as(x)
                elif isinstance(m, nn.GroupNorm):
                    x = F.group_norm(hi, m.num_groups, w, b, m.eps).type_as(x)
                else:
                    x = m(x)
        return x

    def get_out_seq_lens_tensor(self, lengths):  # :365-374
        out = lengths.clone()
        for _, k, s in self.specs:
            out = ((out.float() - (k - 1) - 1) / s + 1).floor().long()
        return out


class SpeechEncoderPrenet(nn.Module):
    """modules/speech_encoder_prenet.py:57-275: conv front-end, mean-square feature penalty, LayerNorm(512), padding
    mask down-sampling, Linear 512 -> d, dropout, HuBERT-style time / channel masking, weight-normed grouped
    positional conv (+ SamePad + GELU) and sinusoidal positions of the padding mask.

    The reference draws the mask positions with numpy on the host (compute_mask_indices); here they are inputs
    (`mask_indices` [B,T] bool, `mask_channel_indices` [B,C] bool) so that the oracle and the device path can be fed
    the same draw."""

    def __init__(self, args):
        super().__init__()
        self.args = args
        layers = list(getattr(args, "conv_feature_layers", CONV_FEATURE_LAYERS))  # eval(args.conv_feature_layers), :80
        self.embed = layers[-1][0]
        self.feature_extractor = ConvFeatureExtractionModel(layers, args.extractor_mode, args.conv_bias)
        d = args.encoder_embed_dim
        self.post_extract_proj = nn.Linear(self.embed, d) if self.embed != d else None
        self.feature_grad_mult = args.feature_grad_mult
        self.dropout_p = args.dropout
        self.use_conv_pos, self.use_sinc_pos = args.use_conv_pos, args.use_sinc_pos
        if self.use_conv_pos:
            self.layer_norm = nn.LayerNorm(self.embed)
            conv = nn.Conv1d(d, d, kernel_size=args.conv_pos, padding=args.conv_pos // 2, groups=args.conv_pos_groups)
            nn.init.normal_(conv.weight, mean=0, std=math.sqrt(4.0 / (args.conv_pos * d)))
            nn.init.constant_(conv.bias, 0)
            # nn.utils.weight_norm(conv, name="weight", dim=2): g has shape [1, 1, K], v the weight's
            self.pos_conv_g = nn.Parameter(conv.weight.detach().norm(dim=(0, 1), keepdim=True))
            self.pos_conv_v = nn.Parameter(conv.weight.detach().clone())
            self.pos_conv_bias = nn.Parameter(conv.bias.detach().clone())
            self.conv_pos, self.conv_pos_groups = args.conv_pos, args.conv_pos_groups
        if self.use_sinc_pos:
            self.embed_positions = SinusoidalPositionalEmbedding(d, 1)  # padding_idx = 1 (:75)
        self.mask_emb = nn.Parameter(torch.empty(d).uniform_())

    def pos_conv_weight(self):
        v = self.pos_conv_v
        return self.pos_conv_g * v / v.norm(dim=(0, 1), keepdim=True)

    def forward_padding_mask(self, features, padding_mask):  # :219-229
        extra = padding_mask.size(1) % features.size(1)
        if extra > 0:
            padding_mask = padding_mask[:, :-extra]
        return padding_mask.view(padding_mask.size(0), features.size(1), -1).all(-1)

    def forward(self, source, padding_mask=None, mask_indices=None, mask_channel_indices=None):
        if self.feature_grad_mult > 0:
            x = self.feature_extractor(source)
            if self.feature_grad_mult != 1.0:  # GradMultiply: identity forward, gradient scaled
                x = x * self.feature_grad_mult + x.detach() * (1.0 - self.feature_grad_mult)
        else:
            with torch.no_grad():
                x = self.feature_extractor(source)
        features_pen = x.float().pow(2).mean()  # :172
        x = self.layer_norm(x.transpose(1, 2))  # [B, T, 512]
        enc_padding_mask = self.forward_padding_mask(x, padding_mask) if padding_mask is not None else None
        if self.post_extract_proj is not None:
            x = self.post_extract_proj(x)
        x = F.dropout(x, self.dropout_p, self.training)
        if mask_indices is not None:  # :230-251
            x = x.clone()
            x[mask_indices] = self.mask_emb.to(x.dtype)
        if mask_channel_indices is not None:  # :253-271
            x = x.masked_fill(mask_channel_indices.unsqueeze(1).expand(-1, x.size(1), -1), 0.0)
        if self.use_conv_pos:  # :186-190
            pos = F.conv1d(x.transpose(1, 2), self.pos_conv_weight(), self.pos_conv_bias, padding=self.conv_pos // 2,
                           groups=self.conv_pos_groups)
            if self.conv_pos % 2 == 0:
                pos = pos[:, :, :-1]  # SamePad
            x = x + F.gelu(pos).transpose(1, 2)
        if self.use_sinc_pos:  # :196-198
            pm = enc_padding_mask if enc_padding_mask is not None else torch.zeros(x.shape[:2], dtype=torch.bool)
            x = x + self.embed_positions(pm).to(x.dtype)
        return x, enc_padding_mask, features_pen


# ------------------------------------------------------------------------------------------------ text decoder pre/post
class TextDecoderPrenet(nn.Module):
    """modules/text_decoder_prenet.py:29-124 (no quant noise, no incremental state): scale * E[tok] + sinusoidal
    positions (fairseq layout), optional LayerNorm, dropout; padding mask only if a pad is present (:90-93)."""

    def __init__(self, embed_tokens, args):
        super().__init__()
        d = args.decoder_embed_dim
        self.embed_tokens = embed_tokens
        self.padding_idx = embed_tokens.padding_idx
        self.embed_scale = 1.0 if args.no_scale_embedding else math.sqrt(d)
        self.embed_positions = (None if args.no_token_positional_embeddings
                                else SinusoidalPositionalEmbedding(d, self.padding_idx))
        self.layernorm_embedding = nn.LayerNorm(d) if getattr(args, "layernorm_embedding", False) else None
        self.dropout_p = args.dropout

    def forward(self, prev_output_tokens):
        x_mask = prev_output_tokens.eq(self.padding_idx) if prev_output_tokens.eq(self.padding_idx).any() else None
        x = self.embed_scale * self.embed_tokens(prev_output_tokens)
        if self.embed_positions is not None:
            x = x + self.embed_positions(prev_output_tokens).to(x.dtype)
        if self.layernorm_embedding is not None:
            x = self.layernorm_embedding(x)
        return F.dropout(x, self.dropout_p, self.training), x_mask


class TextDecoderPostnet(nn.Module):
    """modules/text_decoder_postnet.py:21-93: output projection, tied to the embedding under
    --share-input-output-embed, else Linear(d, V, bias=False) ~ N(0, d^-0.5)."""

    def __init__(self, embed_tokens, vocab_size, args):
        super().__init__()
        d = args.decoder_output_dim if hasattr(args, "decoder_output_dim") else args.decoder_embed_dim
        self.output_projection = nn.Linear(d, vocab_size, bias=False)
        if args.share_input_output_embed:
            self.output_projection.weight = embed_tokens.weight
        else:
            nn.init.normal_(self.output_projection.weight, mean=0, std=d ** -0.5)

    def forward(self, x):
        return self.output_projection(x)


# ------------------------------------------------------------------------------------------------ model
class T5TransformerModelASROracle(nn.Module):
    """models/speecht5.py:47-116 + the s2t branch of forward (:786-963): speech prenet -> shared encoder (with the CTC
    head, encoder.py:101-111,173-179) -> text decoder prenet -> decoder -> vocabulary projection. Returns the
    reference's ((logits [B,T,V], None), encoder_output)."""

    def __init__(self, args, vocab_size=81, padding_idx=1):
        super().__init__()
        self.args = args
        d = args.encoder_embed_dim

        def embedding():
            m = nn.Embedding(vocab_size, d, padding_idx=padding_idx)
            nn.init.normal_(m.weight, mean=0, std=d ** -0.5)
            nn.init.constant_(m.weight[padding_idx], 0)
            return m

        dec_embed = embedding()
        enc_embed = dec_embed if args.share_input_output_embed else embedding()
        self.encoder = TransformerEncoder(args, vocab_size, enc_embed)
        self.decoder = TransformerDecoder(args)
        self.speech_encoder_prenet = SpeechEncoderPrenet(args)
        self.text_decoder_prenet = TextDecoderPrenet(dec_embed, args)
        self.text_decoder_postnet = TextDecoderPostnet(dec_embed, vocab_size, args)
        if args.bert_init:
            self.apply(init_bert_params)

    def forward(self, source=None, padding_mask=None, prev_output_tokens=None, mask_indices=None,
                mask_channel_indices=None, task_name="s2t", **unused):
        x, enc_pad, features_pen = self.speech_encoder_prenet(source, padding_mask, mask_indices, mask_channel_indices)
        encoder_output = self.encoder(x, enc_pad)
        encoder_output["features_pen"] = features_pen
        dec_in, tgt_mask = self.text_decoder_prenet(prev_output_tokens)
        decoder_output, _ = self.decoder(dec_in, tgt_mask, encoder_output, alignment_layer=None)
        return (self.text_decoder_postnet(decoder_output), None), encoder_output

    def get_normalized_probs_for_ctc(self, encoder_output, log_probs=True):  # models/speecht5.py:742-749
        logits = encoder_output["encoder_out_for_ctc"][0].float()
        return F.log_softmax(logits, dim=-1) if log_probs else F.softmax(logits, dim=-1)


# ------------------------------------------------------------------------------------------------ criterion
def label_smoothed_nll_loss(lprobs, target, epsilon, ignore_index):
    """criterions/speech_to_text_loss.py:93-110 (note the reference's (1 - eps - eps_i) weighting)."""
    target = target.unsqueeze(-1)
    nll = -lprobs.gather(dim=-1, index=target)
    smooth = -lprobs.sum(dim=-1, keepdim=True)
    pad = target.eq(ignore_index)
    nll = nll.masked_fill(pad, 0.0).sum()
    smooth = smooth.masked_fill(pad, 0.0).sum()
    eps_i = epsilon / (lprobs.size(-1) - 1)
    return (1.0 - epsilon - eps_i) * nll + eps_i * smooth, nll


def asr_loss(model, sample, ce_weight=0.5, ctc_weight=0.5, label_smoothing=0.1, pad_idx=1, eos_idx=2, blank_idx=0):
    """SpeechtoTextLoss.forward (criterions/speech_to_text_loss.py:186-337): label-smoothed NLL on
    log_softmax_fp32(decoder logits) + CTC(sum, zero_infinity) on the encoder head with target_lengths - 1 (:324).
    Returns (loss, ce, ctc, sample_size); sample_size = number of sentences (sentence_avg, the recipe's setting)."""
    (logits, _), enc = model(**sample["net_input"])
    lprobs = F.log_softmax(logits.float(), dim=-1)
    ce, _ = label_smoothed_nll_loss(lprobs.view(-1, lprobs.size(-1)), sample["target"].view(-1), label_smoothing, pad_idx)
    ctc_lp = model.get_normalized_probs_for_ctc(enc, log_probs=True).contiguous()  # [T, B, V]
    if enc["encoder_padding_mask"][0] is not None:
        input_lengths = (~enc["encoder_padding_mask"][0]).long().sum(-1)
    else:
        input_lengths = ctc_lp.new_full((ctc_lp.size(1),), ctc_lp.size(0), dtype=torch.long)
    keep = (sample["target"] != pad_idx) & (sample["target"] != eos_idx)
    targets_flat = sample["target"].masked_select(keep)
    target_lengths = sample["target_lengths"] - 1
    ctc = F.ctc_loss(ctc_lp, targets_flat, input_lengths, target_lengths, blank=blank_idx, reduction="sum",
                     zero_infinity=True)
    loss = ce_weight * ce + ctc_weight * ctc
    return loss, ce, ctc, sample["target"].size(0)


def synthetic_asr_batch(B, n_samples, T_tgt, vocab=81, seed=1, ragged=True, pad=1, eos=2, bos=2):
    """SURVEY 8(d) config 3 shaped batch: waveforms N(0, 0.1^2) with ragged lengths (-> padding_mask), targets
    U{4..V-1} ending in eos, prev_output_tokens = eos-shifted targets (fairseq collater convention,
    data/speech_to_text_dataset.py:191-204)."""
    g = torch.Generator().manual_seed(seed)
    wav = torch.randn(B, n_samples, generator=g) * 0.1
    lens = torch.full((B,), n_samples, dtype=torch.long)
    tlen = torch.full((B,), T_tgt, dtype=torch.long)
    if ragged and B > 1:
        lens = torch.randint(int(0.8 * n_samples), n_samples + 1, (B,), generator=g)
        lens[0] = n_samples
        tlen = torch.randint(max(2, T_tgt // 2), T_tgt + 1, (B,), generator=g)
        tlen[0] = T_tgt
    padding_mask = torch.arange(n_samples)[None, :] >= lens[:, None]
    wav = wav.masked_fill(padding_mask, 0.0)
    target = torch.full((B, T_tgt), pad, dtype=torch.long)
    for b in range(B):
        n = int(tlen[b])
        target[b, : n - 1] = torch.randint(4, vocab, (n - 1,), generator=g)
        target[b, n - 1] = eos
    prev = torch.full_like(target, pad)
    prev[:, 0] = bos
    for b in range(B):
        n = int(tlen[b])
        prev[b, 1:n] = target[b, : n - 1]
    return {"net_input": {"source": wav, "padding_mask": padding_mask, "prev_output_tokens": prev, "task_name": "s2t"},
            "target": target, "target_lengths": tlen, "ntokens": int(tlen.sum())}


def compute_mask_indices_static(B, T, padding_mask, mask_prob, mask_length, rng, min_masks=2):
    """fairseq/data/data_utils.py compute_mask_indices, mask_type "static", overlapping spans allowed, as called by
    apply_hubert_mask (speech_encoder_prenet.py:236-248): per row num_mask = int(mask_prob * sz / mask_length +
    rand()), at least min_masks, span starts sampled without replacement, rows truncated to the common minimum."""
    mask = np.full((B, T), False)
    idcs = []
    for b in range(B):
        sz = T - int(padding_mask[b].long().sum()) if padding_mask is not None else T
        num_mask = max(min_masks, int(mask_prob * sz / float(mask_length) + rng.random()))
        if sz - mask_length <= num_mask:
            mask_len = sz - num_mask - 1 if sz - num_mask - 1 > 0 else 1  # (degenerate short rows)
        else:
            mask_len = mask_length
        starts = rng.choice(sz - mask_len, num_mask, replace=False)
        idc = np.asarray([s + o for s in starts for o in range(mask_len)])
        idcs.append(np.unique(idc[idc < sz]))
    min_len = min(len(m) for m in idcs)
    for b, idc in enumerate(idcs):
        if len(idc) > min_len:
            idc = rng.choice(idc, min_len, replace=False)
        mask[b, idc] = True
    return torch.from_numpy(mask)


# ------------------------------------------------------------------------------------------------ greedy decode (row 21)
@torch.no_grad()
def greedy_decode(model, source, padding_mask=None, max_len_a=0.0, max_len_b=200, min_len=1, max_positions=600,
                  pad=1, eos=2, unk=3, blank=0, mask_idx=None, unk_penalty=0.0, temperature=1.0):
    """speecht5/sequence_generator.py:207-655 with beam 1, ctc_weight 0, no LM fusion (the `generate.py` greedy
    setting the north-star parity statement refers to: token ids must match bit for bit).

    Encoder once (speecht5.py:1133-1149 forward_encoder); per step the decoder on the prefix, log_softmax / T
    (:1151-1164), then the reference's masking order (:430-446): eos forbidden before min_len, NaN -> -inf, pad never,
    unk penalty, CTC blank (and mask symbol) never, only eos at step >= max_len; argmax. The prefix starts with eos
    (bos_token None, :303). max_len = min(int(a * src_len + b), max_positions - 1) where src_len is the PADDED source
    length (waveform samples for speech input, :249,262-265). Returns a list of 1-D token tensors ending in eos."""
    B = source.size(0)
    src_len = source.size(1)
    max_len = min(int(max_len_a * src_len + max_len_b), max_positions - 1)
    assert min_len <= max_len
    x, enc_pad, _ = model.speech_encoder_prenet(source, padding_mask, None, None)
    enc = model.encoder(x, enc_pad)
    tokens = torch.full((B, max_len + 2), pad, dtype=torch.long)
    tokens[:, 0] = eos
    done = [False] * B
    out = [None] * B
    for step in range(max_len + 1):
        dec_in, tgt_mask = model.text_decoder_prenet(tokens[:, : step + 1])
        z, _ = model.decoder(dec_in, tgt_mask, enc, alignment_layer=None)
        logits = model.text_decoder_postnet(z[:, -1:, :])[:, -1, :]
        lprobs = F.log_softmax(logits.float() / temperature, dim=-1)
        if step < min_len:
            lprobs[:, eos] = -math.inf
        lprobs[lprobs != lprobs] = -math.inf
        lprobs[:, pad] = -math.inf
        lprobs[:, unk] -= unk_penalty
        lprobs[:, blank] = -math.inf
        if mask_idx is not None and mask_idx != unk:
            lprobs[:, mask_idx] = -math.inf
        if step >= max_len:
            lprobs[:, :eos] = -math.inf
            lprobs[:, eos + 1:] = -math.inf
        nxt = lprobs.argmax(dim=-1)
        tokens[:, step + 1] = nxt
        for b in range(B):
            if not done[b] and int(nxt[b]) == eos:
                done[b] = True
                out[b] = tokens[b, 1: step + 2].clone()
        if all(done):
            break
    return out


# ------------------------------------------------------------------------------------------------ text in / text out
class T5TransformerModelT2TOracle(nn.Module):
    """models/speecht5.py:786-963, text input + text output (the BART-style text branch of pre-training and the MT-like
    fine-tunes): text encoder prenet (espnet scaled positional encoding) -> shared encoder -> text decoder prenet ->
    decoder -> vocabulary projection. Returns the reference's ((logits, None), codebook_out = {}, encoder_output)."""

    def __init__(self, args, vocab_size=81, padding_idx=1):
        super().__init__()
        from .speecht5_oracle import TextEncoderPrenet
        self.args = args
        d = args.encoder_embed_dim

        def embedding():
            m = nn.Embedding(vocab_size, d, padding_idx=padding_idx)
            nn.init.normal_(m.weight, mean=0, std=d ** -0.5)
            nn.init.constant_(m.weight[padding_idx], 0)
            return m

        dec_embed = embedding()
        enc_embed = dec_embed if args.share_input_output_embed else embedding()
        self.encoder = TransformerEncoder(args, vocab_size, enc_embed)
        self.decoder = TransformerDecoder(args)
        self.text_encoder_prenet = TextEncoderPrenet(enc_embed, args)
        self.text_decoder_prenet = TextDecoderPrenet(dec_embed, args)
        self.text_decoder_postnet = TextDecoderPostnet(dec_embed, vocab_size, args)
        if args.bert_init:
            self.apply(init_bert_params)

    def forward(self, src_tokens=None, prev_output_tokens=None, **unused):
        encoder_input, encoder_padding_mask = self.text_encoder_prenet(src_tokens)
        encoder_output = self.encoder(encoder_input, encoder_padding_mask)
        dec_in, tgt_mask = self.text_decoder_prenet(prev_output_tokens)
        decoder_output, _ = self.decoder(dec_in, tgt_mask, encoder_output, alignment_layer=None)
        return (self.text_decoder_postnet(decoder_output), None), {}, encoder_output


def reference_to_oracle_keys(sd):
    """Rename a state dict of the REFERENCE model (checkpoint key layout) to this oracle's few differing names:
    the weight-normed positional conv lives at `pos_conv.0.{weight_g,weight_v,bias}` in the reference
    (speech_encoder_prenet.py:105-119) and the layer_norm-mode extractor wraps its norm as
    Sequential(TransposeLast, Fp32LayerNorm, TransposeLast) -> `conv_layers.{i}.2.1.*` (:308-318)."""
    import re
    out = {}
    for k, v in sd.items():
        k = k.replace("pos_conv.0.weight_g", "pos_conv_g").replace("pos_conv.0.weight_v", "pos_conv_v")
        k = k.replace("pos_conv.0.bias", "pos_conv_bias")
        k = re.sub(r"(conv_layers\.\d+\.2)\.1\.", r"\1.", k)
        out[k] = v
    return out
