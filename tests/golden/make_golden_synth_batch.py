"""Generator of tests/golden/ref_synth_batch_tiny.npz: the REFERENCE's own batch-1 generate_speech
(models/speecht5.py:1188-1249) on every utterance of two batches, the pin of generate_speech_batch:
  * TTS: 4 texts of 7 / 5 / 3 / 9 tokens, each with its own x-vector;
  * VC: the 3 waveforms of make_golden_vc.py (12 / 8 / 5 conv frames), each with its own x-vector.
The model is make_golden_vc.py's (tiny widths, t5_transformer_base_asr structure with relative positions, reduction
factor 2, every dropout off including the decoder prenet's, parameters filled from their NAMES with seed_parameters of
tests/test_ref_pin_cpu.py, seed make_golden_vc.SEED; the reference builds the text prenet for the s2s task too), in
eval mode without an update. Each case adds a stop-logit offset to prob_out.bias (see CASES) so that, between them, the
utterances stop on a stop probability, at their own maxlen, and later than a stop probability because `threshold` was
passed (the quirk that also sets minlenratio and maxlenratio).

Stored: in/tts/{tokens,lengths,spkembs}, in/vc/{source,padding_mask,spkembs}, and <batch>/<case>/<b>/{mel,probs,attn}.

usage: python tests/golden/make_golden_synth_batch.py     (needs the reference tree, see oracle/ref_loader.py)"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import make_golden_vc as mv  # noqa: E402
from speecht5_b200.data import collate_vc  # noqa: E402

OUT = os.path.join(HERE, "ref_synth_batch_tiny.npz")
TEXT_LENS = (7, 5, 3, 9)
# case: (generate_speech kwargs, stop-logit offset per batch)
CASES = {
    "default": ({}, {"tts": -3.0, "vc": -3.0}),       # no probability reaches 0.5: every utterance stops at its maxlen
    "stop": ({}, {"tts": -1.16, "vc": -2.45}),        # stops on a stop probability, the shortest at its maxlen
    "threshold": ({"threshold": 0.9}, {"tts": 2.5, "vc": 2.5}),  # minlen = maxlen: later than the probability
}


def inputs():
    g = torch.Generator().manual_seed(17)
    tokens = torch.ones(len(TEXT_LENS), max(TEXT_LENS), dtype=torch.long)  # padding index 1
    for b, n in enumerate(TEXT_LENS):
        tokens[b, :n] = torch.randint(4, mv.VOCAB, (n,), generator=g)
    tts_spk = torch.randn(len(TEXT_LENS), 512, generator=g)
    ni = collate_vc(mv.items(), 2)["net_input"]
    return {"tts": dict(tokens=tokens, lengths=torch.tensor(TEXT_LENS), spkembs=tts_spk),
            "vc": dict(source=ni["source"], padding_mask=ni["padding_mask"], spkembs=ni["spkembs"])}


def utterance_kwargs(batch, inp, b):
    """generate_speech inputs of utterance b alone (padding stripped)."""
    if batch == "tts":
        n = int(inp["lengths"][b])
        return dict(src_tokens=inp["tokens"][b:b + 1, :n], spkembs=inp["spkembs"][b:b + 1])
    n = int((~inp["padding_mask"][b]).sum())
    return dict(source=inp["source"][b:b + 1, :n], padding_mask=inp["padding_mask"][b:b + 1, :n],
                spkembs=inp["spkembs"][b:b + 1])


def main(path=OUT):
    _, _, model = mv.build()
    model.eval()
    inp = inputs()
    blob = {f"in/{batch}/{k}": v.numpy() for batch, d in inp.items() for k, v in d.items()}
    bias = model.speech_decoder_postnet.prob_out.bias
    with torch.no_grad():
        for case, (kw, offsets) in CASES.items():
            for batch, d in inp.items():
                bias.add_(offsets[batch])
                for b in range(d["spkembs"].shape[0]):
                    mel, probs, att = model.generate_speech(**utterance_kwargs(batch, d, b), **kw)
                    blob[f"{batch}/{case}/{b}/mel"] = mel.numpy()
                    blob[f"{batch}/{case}/{b}/probs"] = probs.numpy()
                    blob[f"{batch}/{case}/{b}/attn"] = att.numpy()
                bias.sub_(offsets[batch])
    if path is not None:
        np.savez_compressed(path, **blob)
        print(path, os.path.getsize(path), "bytes")
    return blob


if __name__ == "__main__":
    blob = main()
    for k in sorted(blob):
        if k.endswith("/probs"):
            p = blob[k].reshape(-1, 2)
            hit = np.nonzero((p >= 0.5).any(1))[0]
            print(k, "steps", p.shape[0], "first prob >= 0.5 at step", (hit[0] + 1) if len(hit) else None)
