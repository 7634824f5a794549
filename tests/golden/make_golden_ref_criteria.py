"""Generator of tests/golden/ref_criteria_dict.npz: what the reference's OWN pre-training criteria and fairseq
Dictionary return on the inputs of tests/test_ref_pin_cpu.py (criteria: loss, sample size, logging values, the gradients
on the model outputs of _PretrainStub; Dictionary: indices, lookups, appended symbols, id -> text). The tests compare the
product against these vectors, so they run without the reference tree.

usage: python tests/golden/make_golden_ref_criteria.py     (needs the reference tree, see oracle/ref_loader.py)"""
import importlib
import json
import os
import sys
import tempfile

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

OUT = os.path.join(HERE, "ref_criteria_dict.npz")


def _num(v):
    return float(v.item()) if torch.is_tensor(v) else float(v)


def main():
    rl.load()
    meta, arrays = {"speech": {}, "text": {}}, {}
    ref_mod = importlib.import_module("speecht5.criterions.speech_pretrain_criterion")
    task = rl.RefTask(mg.VOCAB, "pretrain")
    for dec_weight, nomask, weights in t.SPEECH_CASES:
        key = t.speech_case_key(dec_weight, nomask, weights)
        kw = dict(pred_masked_weight=1.0, pred_nomask_weight=nomask, loss_weights=None if weights is None else list(weights),
                  log_keys=["temp"], hubert_weight=0.7, dec_weight=dec_weight)
        ms = t._PretrainStub(4)
        loss, n, log = ref_mod.SpeechPretrainCriterion(task, True, **kw)(ms, t._speech_pretrain_sample())
        loss.backward()
        meta["speech"][key] = {"loss": _num(loss), "n": _num(n), "log": {k: _num(v) for k, v in log.items()},
                               "only_hubert": bool(ms.calls[0].get("only_hubert", False)),
                               "grads": [name for name, p in ms.named_parameters() if p.grad is not None]}
        for name, p in ms.named_parameters():
            if p.grad is not None:
                arrays[f"speech/{key}/{name}"] = p.grad.numpy()
    ref_mod = importlib.import_module("speecht5.criterions.text_pretrain_criterion")
    for sentence_avg, weights in t.TEXT_CASES:
        key = t.text_case_key(sentence_avg, weights)
        ms = t._PretrainStub(6, text=True)
        loss, n, log = ref_mod.TextPretrainCriterion(task, sentence_avg, 0.9, list(weights))(ms, t._text_pretrain_sample(task))
        loss.backward()
        meta["text"][key] = {"loss": _num(loss), "n": _num(n), "log": {k: _num(v) for k, v in log.items()},
                             "pp_grad": None if ms.pp.grad is None else _num(ms.pp.grad)}
        arrays[f"text/{key}/logits"] = ms.logits.grad.numpy()
    Ref = t._reference_dictionary_class()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "dict.txt")
        with open(path, "w", encoding="utf-8") as fh:
            fh.write(t.dict_file_text())
        meta["dictionary"] = t.dictionary_observations(Ref.load(path))
    np.savez_compressed(OUT, meta=np.array(json.dumps(meta, sort_keys=True)), **arrays)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
