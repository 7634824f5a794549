"""Generator of tests/golden/ref_pins.npz: what the reference's OWN code returns for the pins of tests/test_ref_pin_cpu.py
that used to need the reference tree at test time -- the encoder at ASR lengths and the conv feature extractor at real
width (sampled outputs, parameters filled by name with seed_parameters), generate_speech on a tiny model (the mel), the
meters of SpeechT5Criterion.reduce_metrics, the arch presets, the criterion dataclass defaults and the model / task
command-line option tables.

usage: python tests/golden/make_golden_ref_pins.py     (needs the reference tree, see oracle/ref_loader.py)"""
import importlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)

import make_golden_from_ref as mg  # noqa: E402
import test_ref_pin_cpu as t  # noqa: E402
from oracle import ref_loader as rl  # noqa: E402

OUT = os.path.join(HERE, "ref_pins.npz")


def main():
    ns = rl.load()
    meta, arrays = {}, {}
    # encoder at T = 199 / 499
    enc = ns.encoder.TransformerEncoder(rl.reference_args(**t.ENC_OVER), rl.RefDictionary(mg.VOCAB), None).eval()
    t.seed_parameters(enc, 3)
    meta["encoder_params"] = sorted(n for n, _ in enc.named_parameters())
    for T in (199, 499):
        x, pad = t.encoder_input(T)
        with torch.no_grad():
            out = enc(x, pad)
        arrays[f"encoder/{T}/out"] = t.output_sample(out["encoder_out"][0]).numpy()
        arrays[f"encoder/{T}/ctc"] = t.output_sample(out["encoder_out_for_ctc"][0]).numpy()
    # conv feature extractor, 512 channels, both modes
    from oracle.speecht5_oracle_asr import CONV_FEATURE_LAYERS
    x = t.conv_extractor_input()
    for mode in ("default", "layer_norm"):
        ref = ns.speech_encoder_prenet.ConvFeatureExtractionModel(CONV_FEATURE_LAYERS, 0.0, mode, False).eval()
        t.seed_parameters(ref, 5)
        meta[f"conv/{mode}/shapes"] = {n: list(p.shape) for n, p in ref.named_parameters()}
        with torch.no_grad():
            arrays[f"conv/{mode}/out"] = t.output_sample(ref(x)).numpy()
    # generate_speech on the tiny t2s model
    ref = rl.build_reference_model(rl.reference_args(**t.GEN_OVER), rl.RefTask(mg.VOCAB, "t2s")).eval()
    t.seed_parameters(ref, 21)
    meta["generate_params"] = sorted(n for n, _ in ref.named_parameters())
    toks, spk = t.generate_speech_inputs()
    with torch.no_grad():
        mel = ref.generate_speech(source=None, src_tokens=toks, spkembs=spk, threshold=0.5, minlenratio=0.0, maxlenratio=2.0)
    arrays["generate/mel"] = mel[0].numpy()
    # reduce_metrics
    crit = importlib.import_module("speecht5.criterions.speecht5_criterion")
    ns.metrics.logged.clear()
    ns.metrics.derived.clear()
    crit.SpeechT5Criterion.reduce_metrics(t.REDUCE_LOGS)
    meta["reduce_metrics"] = {"logged": {k: float(v) for k, v in ns.metrics.logged.items()},
                              "derived": sorted(ns.metrics.derived)}
    # arch presets, criterion defaults, option tables
    meta["arch"] = {a: t.jsonable(vars(rl.reference_args(arch=a))) for a in t.ARCHS}
    meta["criterion_defaults"] = t.jsonable(t.dataclass_defaults(crit.SpeechT5CriterionConfig))
    meta["model_add_args"] = t.jsonable(t.add_args_table(ns.T5TransformerModel)[1])
    with open(os.path.join(rl.ST5, "speecht5", "tasks", "speecht5.py")) as fh:
        meta["task_add_args"] = t.jsonable(t.task_add_argument_calls(fh.read()))
    np.savez_compressed(OUT, meta=np.array(json.dumps(meta, sort_keys=True)), **arrays)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
