"""TEST INFRASTRUCTURE (never imported by the product path): the reference's language model for LM-fusion fixtures
(`tests/golden/make_golden_beam_lm.py`), loaded unmodified on top of `oracle/ref_loader.py` (same machinery: reference
files executed by path under their real module names, single definitions AST-extracted from files too entangled to
execute, infrastructure stubbed). Needs the reference tree (`ref_loader.available()`)."""
import os
import sys
import types

from oracle import ref_loader as rl

_loaded = {}


def load_lm():
    """fairseq's transformer_lm, unmodified: `TransformerLanguageModel` and `base_lm_architecture`
    (fairseq/models/transformer_lm.py) and `TransformerDecoder` (fairseq/models/transformer.py), AST-extracted like
    `Embedding` / `Linear`, on the real `fairseq/modules/transformer_layer.py` and `fairseq/modules/multihead_attention.py`.

    SpeechT5's modules were imported against the `fairseq.modules.multihead_attention` stub of ref_loader (an
    isinstance / annotation target); the real module is executed here for the LM's layers and the stub is put back
    afterwards, so the SpeechT5 classes see what they saw before."""
    if "lm" in _loaded:
        return _loaded["lm"]
    import math
    import typing
    import torch
    import torch.nn as nn
    ns = rl.load()
    fm, fmod = sys.modules["fairseq.modules"], sys.modules["fairseq.models"]
    stub_mod, stub_cls = sys.modules["fairseq.modules.multihead_attention"], fm.MultiheadAttention
    try:
        mha = rl._exec_file("fairseq.modules.multihead_attention", os.path.join(rl.FAIRSEQ, "modules", "multihead_attention.py"))
        fm.MultiheadAttention = mha.MultiheadAttention
        tl = rl._exec_file("fairseq.modules.transformer_layer", os.path.join(rl.FAIRSEQ, "modules", "transformer_layer.py"))
    finally:
        sys.modules["fairseq.modules.multihead_attention"] = stub_mod
        fm.multihead_attention, fm.MultiheadAttention = stub_mod, stub_cls
    tr = sys.modules["fairseq.models.transformer"]
    tr.__dict__.update(
        math=math, utils=sys.modules["fairseq.utils"], Tensor=torch.Tensor, Any=typing.Any, Dict=typing.Dict,
        List=typing.List, Optional=typing.Optional, Tuple=typing.Tuple,
        FairseqIncrementalDecoder=fmod.FairseqIncrementalDecoder, FairseqDropout=fm.FairseqDropout,
        LayerDropModuleList=fm.LayerDropModuleList, PositionalEmbedding=fm.PositionalEmbedding,
        AdaptiveSoftmax=fm.AdaptiveSoftmax, TransformerDecoderLayer=tl.TransformerDecoderLayer,
        apply_quant_noise_=sys.modules["fairseq.modules.quant_noise"].quant_noise,
        checkpoint_wrapper=sys.modules["fairseq.modules.checkpoint_activations"].checkpoint_wrapper,
        fsdp_wrap=sys.modules["fairseq.distributed"].fsdp_wrap, DEFAULT_MIN_PARAMS_TO_WRAP=int(1e8),
        DEFAULT_MAX_TARGET_POSITIONS=1024)
    rl._extract(os.path.join(rl.FAIRSEQ, "models", "transformer.py"), ["TransformerDecoder"], tr.__dict__, tr.__name__)
    lm_ns = {"nn": nn, "torch": torch, "options": None, "utils": sys.modules["fairseq.utils"],
             "FairseqLanguageModel": fmod.FairseqLanguageModel, "register_model": fmod.register_model,
             "register_model_architecture": fmod.register_model_architecture,
             "TransformerLanguageModelConfig": type("TransformerLanguageModelConfig", (), {}),
             "Embedding": tr.Embedding, "TransformerDecoder": tr.TransformerDecoder, "DEFAULT_MAX_TARGET_POSITIONS": 1024,
             "AdaptiveInput": None, "CharacterTokenEmbedder": None}
    rl._extract(os.path.join(rl.FAIRSEQ, "models", "transformer_lm.py"), ["TransformerLanguageModel", "base_lm_architecture"],
             lm_ns, "fairseq.models.transformer_lm")
    out = types.SimpleNamespace(TransformerLanguageModel=lm_ns["TransformerLanguageModel"],
                                base_lm_architecture=lm_ns["base_lm_architecture"],
                                TransformerDecoder=tr.TransformerDecoder,
                                TransformerDecoderLayer=tl.TransformerDecoderLayer, MultiheadAttention=mha.MultiheadAttention,
                                sequence_generator=ns.sequence_generator)
    _loaded["lm"] = out
    return out
