"""The language model of shallow fusion (`generate.py --lm-path LM --lm-weight W`, speecht5/sequence_generator.py:420-426):
fairseq's `transformer_lm` (fairseq/models/transformer_lm.py:200-362 with the TransformerDecoder of
fairseq/models/transformer.py:637-986, no encoder attention) on this package's kernels.

Built configuration: heads of 64 or 80 channels (80: SpeechT5's own `transformer_lm_t5`, 1280 channels in 16 heads,
whose preset applies when the arguments name that arch), rows up to 2048 channels, pre-LN decoder layers
(base_lm_architecture forces decoder_normalize_before), sinusoidal or learned positions at padding_idx + 1 + i,
embed_scale = sqrt(C) unless no_scale_embedding, an optional final LayerNorm (no_decoder_final_norm), an output
projection tied to the embedding or not, relu or gelu. Adaptive input or softmax,
character embeddings, layernorm_embedding, project_in / project_out dimensions, cross_self_attention and quant noise
raise NotImplementedError when the model is built.

Parameter names are fairseq's (`decoder.embed_tokens.weight`, `decoder.layers.{i}.self_attn.q_proj.weight`, ...), so a
fairseq state dict loads as it is. Beam search runs the model one position per step on a key/value cache
(incremental.BeamGraph); `forward` runs a whole prefix at once."""
import math
from argparse import Namespace

import torch
import torch.nn as nn

from . import ops
from .models.modules.transformer import TransformerDecoderLayer

# fairseq keeps these buffers in a transformer_lm state dict; they carry no weights
_BUFFERS = ("decoder.version", "decoder.embed_positions._float_tensor")
HEAD_DIMS = (64, 80)  # the one-row attention's head widths (80: transformer_lm_t5, 1280 channels in 16 heads)
MAX_DIM = 2048        # the widest LayerNorm row (st5_ln_fwd_wide)

# fairseq's base_lm_architecture (fairseq/models/transformer_lm.py:296-359): an option the arguments lack takes this value
_BASE_LM_DEFAULTS = dict(
    dropout=0.1, attention_dropout=0.0, decoder_embed_dim=512, decoder_ffn_embed_dim=2048, decoder_layers=6,
    decoder_attention_heads=8, adaptive_softmax_cutoff=None, adaptive_softmax_dropout=0, adaptive_softmax_factor=4,
    decoder_learned_pos=False, activation_fn="relu", decoder_layerdrop=0, decoder_layers_to_keep=None, quant_noise_pq=0,
    quant_noise_pq_block_size=8, quant_noise_scalar=0, base_layers=0, base_sublayers=1, base_shuffle=False,
    add_bos_token=False, no_token_positional_embeddings=False, share_decoder_input_output_embed=False,
    character_embeddings=False)
_BASE_LM_DEFAULTS_TAIL = dict(no_decoder_final_norm=False, adaptive_input=False, adaptive_input_factor=4,
                              adaptive_input_cutoff=None, tie_adaptive_weights=False, tie_adaptive_proj=False,
                              no_scale_embedding=False, layernorm_embedding=False, checkpoint_activations=False,
                              offload_activations=False)
# SpeechT5's own LM (speecht5/models/t5_transformer_lm.py: arch transformer_lm_t5), applied before the base defaults
_T5_LM_DEFAULTS = dict(decoder_embed_dim=1280, decoder_ffn_embed_dim=6144, decoder_layers=20, decoder_attention_heads=16,
                       dropout=0.1, attention_dropout=0.1, activation_fn="gelu")


def _fill(args, defaults):
    for k, v in defaults.items():
        if not hasattr(args, k):
            setattr(args, k, v)


def base_lm_architecture(args):
    """Fill `args` in place as fairseq's base_lm_architecture does: options it lacks take their defaults (an option set
    to None stays None), decoder_input_dim / decoder_output_dim follow decoder_embed_dim, the layers are pre-LN, and the
    compatibility rules for old checkpoints (no_tie_adaptive_proj, decoder_final_norm) apply."""
    if hasattr(args, "no_tie_adaptive_proj"):
        args.no_decoder_final_norm = True
        if args.no_tie_adaptive_proj is False:
            args.tie_adaptive_proj = True
    if hasattr(args, "decoder_final_norm"):
        args.no_decoder_final_norm = not args.decoder_final_norm
    _fill(args, _BASE_LM_DEFAULTS)
    _fill(args, dict(decoder_output_dim=args.decoder_embed_dim, decoder_input_dim=args.decoder_embed_dim))
    args.decoder_normalize_before = True
    _fill(args, _BASE_LM_DEFAULTS_TAIL)
    if args.offload_activations:
        args.checkpoint_activations = True
    return args


def transformer_lm_t5(args):
    """The `transformer_lm_t5` preset, in place: 20 layers of 1280 channels, 16 heads of 80, FFN 6144, GELU, dropout
    0.1 for options `args` lacks, then base_lm_architecture."""
    _fill(args, _T5_LM_DEFAULTS)
    return base_lm_architecture(args)


ARCHS = {"transformer_lm": base_lm_architecture, "transformer_lm_t5": transformer_lm_t5}


def _with_arch(args):
    """A copy of `args` filled by its `arch` preset when that is transformer_lm_t5 (other arches: as given, missing
    options taking base_lm_architecture's defaults where they are read)."""
    if getattr(args, "arch", None) != "transformer_lm_t5":
        return args
    return transformer_lm_t5(Namespace(**vars(args)))


def _opt(args, name, default):
    v = getattr(args, name, default)
    return default if v is None else v


def _unbuilt(args):
    """The options of a transformer_lm this module does not build, as (name, value) pairs that are set."""
    C = _opt(args, "decoder_embed_dim", 512)
    checks = [
        ("adaptive_input", bool(_opt(args, "adaptive_input", False))),
        ("adaptive_softmax_cutoff", _opt(args, "adaptive_softmax_cutoff", None) is not None),
        ("tie_adaptive_weights", bool(_opt(args, "tie_adaptive_weights", False))),
        ("character_embeddings", bool(_opt(args, "character_embeddings", False))),
        ("layernorm_embedding", bool(_opt(args, "layernorm_embedding", False))),
        ("decoder_input_dim", _opt(args, "decoder_input_dim", C) != C),
        ("decoder_output_dim", _opt(args, "decoder_output_dim", C) != C),
        ("cross_self_attention", bool(_opt(args, "cross_self_attention", False))),
        ("quant_noise_pq", _opt(args, "quant_noise_pq", 0) != 0),
        ("quant_noise_scalar", _opt(args, "quant_noise_scalar", 0) != 0),
        ("no_token_positional_embeddings", bool(_opt(args, "no_token_positional_embeddings", False))),
    ]
    return [n for n, bad in checks if bad]


def fairseq_sinusoid_table_fp32(num_embeddings, dim, padding_idx):
    """fairseq/modules/sinusoidal_positional_embedding.py:36-58 as fairseq computes it for the LM: in fp32 ([sin | cos]
    halves, divisor half_dim - 1, zero row at padding_idx)."""
    half = dim // 2
    step = math.log(10000) / (half - 1)
    freq = torch.exp(torch.arange(half, dtype=torch.float) * -step)
    ang = torch.arange(num_embeddings, dtype=torch.float).unsqueeze(1) * freq.unsqueeze(0)
    emb = torch.cat([torch.sin(ang), torch.cos(ang)], dim=1).view(num_embeddings, -1)
    if dim % 2 == 1:
        emb = torch.cat([emb, torch.zeros(num_embeddings, 1)], dim=1)
    emb[padding_idx, :] = 0
    return emb


class _Decoder(nn.Module):
    def __init__(self, args, vocab, padding_idx):
        super().__init__()
        C = args.decoder_embed_dim
        self.padding_idx = padding_idx
        self.embed_tokens = nn.Embedding(vocab, C, padding_idx=padding_idx)
        self.learned_pos = bool(args.decoder_learned_pos)
        self.max_target_positions = args.max_target_positions
        if self.learned_pos:  # fairseq/modules/positional_embedding.py: max_positions + padding_idx + 1 rows
            self.embed_positions = nn.Embedding(args.max_target_positions + padding_idx + 1, C, padding_idx=padding_idx)
        self.layers = nn.ModuleList([TransformerDecoderLayer(args, no_encoder_attn=True, head_dims=HEAD_DIMS)
                                     for _ in range(args.decoder_layers)])
        self.layer_norm = None if args.no_decoder_final_norm else nn.LayerNorm(C)
        self.output_projection = nn.Linear(C, vocab, bias=False)
        if args.share_decoder_input_output_embed:
            self.output_projection.weight = self.embed_tokens.weight


class TransformerLM(nn.Module):
    """fairseq's TransformerLanguageModel in evaluation: `decoder` holds its parameters under fairseq's names.
    `args` is an argparse Namespace (or anything with the same attributes) of a transformer_lm; options it leaves out take
    base_lm_architecture's defaults."""

    def __init__(self, args, vocab_size, padding_idx=1):
        super().__init__()
        args = _with_arch(args)
        bad = _unbuilt(args)
        if bad:
            raise NotImplementedError(f"transformer_lm options not built for LM fusion: {', '.join(bad)}")
        C = _opt(args, "decoder_embed_dim", 512)
        H = _opt(args, "decoder_attention_heads", 8)
        if C % H != 0 or C // H not in HEAD_DIMS:
            raise NotImplementedError(f"LM heads of {C / H:g} dimensions: the attention kernels take 64 and 80")
        if C > MAX_DIM:
            raise NotImplementedError(f"LM width {C}: the LayerNorm kernels take at most {MAX_DIM} channels")
        act = _opt(args, "activation_fn", "relu")
        if act not in ("relu", "gelu"):
            raise NotImplementedError(f"LM activation {act!r}: relu and gelu are built")
        self.args = Namespace(
            decoder_embed_dim=C, decoder_attention_heads=H, decoder_ffn_embed_dim=_opt(args, "decoder_ffn_embed_dim", 2048),
            decoder_layers=_opt(args, "decoder_layers", 6), activation_fn=act, decoder_normalize_before=True,
            dropout=0.0, attention_dropout=0.0, activation_dropout=0.0, relu_dropout=0.0,
            decoder_learned_pos=bool(_opt(args, "decoder_learned_pos", False)),
            max_target_positions=int(_opt(args, "max_target_positions", None) or _opt(args, "tokens_per_sample", 1024)),
            no_decoder_final_norm=bool(_opt(args, "no_decoder_final_norm", False)),
            share_decoder_input_output_embed=bool(_opt(args, "share_decoder_input_output_embed", False)),
            no_scale_embedding=bool(_opt(args, "no_scale_embedding", False)))
        self.decoder = _Decoder(self.args, int(vocab_size), int(padding_idx))
        self.padding_idx = int(padding_idx)
        self.vocab_size = int(vocab_size)
        self.embed_scale = 1.0 if self.args.no_scale_embedding else math.sqrt(C)
        self.register_buffer("_unit", torch.ones(()), persistent=False)
        self.eval()

    # ------------------------------------------------------------------------------------------------ construction
    @classmethod
    def from_fairseq(cls, module):
        """The model object fairseq's generate.py passes as `lm_model` (a TransformerLanguageModel)."""
        if isinstance(module, cls):
            return module
        dec = module.decoder
        args = getattr(module, "args", None) or getattr(dec, "args", None)
        if args is None:
            raise ValueError("from_fairseq: the module carries no transformer_lm arguments (.args)")
        if getattr(dec, "adaptive_softmax", None) is not None:
            raise NotImplementedError("transformer_lm options not built for LM fusion: adaptive_softmax_cutoff")
        lm = cls(args, dec.embed_tokens.num_embeddings, dec.padding_idx)
        lm.load_fairseq_state(module.state_dict())
        return lm.to(dec.embed_tokens.weight.device)

    def load_fairseq_state(self, state):
        state = {k: v for k, v in state.items() if k not in _BUFFERS}
        if self.args.share_decoder_input_output_embed:
            state.setdefault("decoder.output_projection.weight", state["decoder.embed_tokens.weight"])
        self.load_state_dict(state, strict=True)

    # ------------------------------------------------------------------------------------------------ evaluation
    def positions(self, n, device):
        """Position rows of the first n tokens (positions padding_idx + 1 + i), fp32 [n, C]."""
        p = self.padding_idx + 1
        if self.decoder.learned_pos:
            W = self.decoder.embed_positions.weight
            if W.shape[0] < p + n:
                raise NotImplementedError(f"learned LM positions cover {W.shape[0] - p} tokens, {n} are needed")
            return W.detach()[p:p + n].float().to(device)
        return fairseq_sinusoid_table_fp32(p + n, self.args.decoder_embed_dim, self.padding_idx)[p:].to(device)

    def scaled_embedding(self):
        """embed_scale * E in fp32 (the product fairseq forms), for the embedding + position kernel at alpha 1."""
        return (self.embed_scale * self.decoder.embed_tokens.weight.detach().float()).contiguous()

    def output_layer(self, x):
        return ops.linear(x, self.decoder.output_projection.weight, (), out_dtype=torch.float32)

    @torch.no_grad()
    def forward(self, tokens):
        """tokens [B, T] without padding -> logits [B, T, V] fp32 (causal; every position sees its prefix)."""
        assert not self.training
        x = ops.scaled_posenc(self.positions(tokens.shape[1], tokens.device), self._unit, 0.0,
                              tokens=tokens.contiguous(), emb=self.scaled_embedding(), padding_idx=self.padding_idx)
        for layer in self.decoder.layers:
            x, _, _ = layer(x, causal=True)
        if self.decoder.layer_norm is not None:
            x = ops.residual_layer_norm(x, None, self.decoder.layer_norm)
        return self.output_layer(x)

    def log_probs(self, tokens):
        """get_normalized_probs(log_probs=True): the fp32 log-softmax of forward(tokens)."""
        return torch.log_softmax(self.forward(tokens).float(), dim=-1)


def _args_of(state):
    args = state.get("args")
    if args is None:
        cfg = state.get("cfg")
        args = cfg["model"] if cfg is not None else None
    if args is None:
        raise ValueError("load_lm: the checkpoint holds neither 'args' nor cfg['model']")
    if isinstance(args, dict):
        args = Namespace(**args)
    return args


def load_lm(path, device=None):
    """A fairseq transformer_lm checkpoint file ({"model": state dict, "args": Namespace} or {"cfg": {"model": ...}})."""
    state = torch.load(path, map_location="cpu", weights_only=False)
    model, args = state["model"], _args_of(state)
    lm = TransformerLM(args, model["decoder.embed_tokens.weight"].shape[0], _opt(args, "padding_idx", 1))
    lm.load_fairseq_state(model)
    return lm.to(device) if device is not None else lm
