"""Generator of tests/golden/ref_sid_tiny.npz: the REFERENCE's own speaker-identification update (T5TransformerModel with
t5_task s2c, models/speecht5.py:805-810, 836-842, 896-897, 925-932, its SpeakerDecoderPostnet, and SpeechtoTextLoss with
label smoothing 0.1 through speecht5_criterion.py:113) on tiny widths, plus its eval-mode generate_class (:1171-1186).

Cases (prefix of every key):
  recipe   the fine-tuning recipe's head: no pooling BN, no embedding post-net, softmax, decoder pooling
  defaults the arch defaults: BN pooling, embedding projection + BN, softmax, ENCODER pooling
  aam      aamsoftmax m 0.2 s 30 with target_list (margin in training), one row's target cosine forced below th
  am       amsoftmax m 0.2 s 30 with target_list
All cases run on one padded batch (batch/in/<net input>). Trunk weights are not stored: both sides fill every parameter
from its NAME (seed_parameters of tests/test_ref_pin_cpu.py, seed SEED). Stored per case: head/<speaker head parameter
or buffer> (after the run: the margin cases overwrite one class row, BatchNorm keeps its running statistics), keys (the
reference model's state-dict key -> shape table), sample/target, out/head_input (what the head received), out/logits,
out/embed, loss [loss, nll_loss, n_correct, total, sample_size, ntokens], grad/<param>, out/pred (generate_class).

usage: python tests/golden/make_golden_sid.py     (needs the reference tree, see oracle/ref_loader.py)"""
import json
import os
import sys
from argparse import Namespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import make_golden_from_ref as mg  # noqa: E402
from oracle import ref_loader as rl  # noqa: E402
from speecht5_b200.data import synthetic_sid_batch  # noqa: E402
from test_ref_pin_cpu import seed_parameters  # noqa: E402

OUT = os.path.join(HERE, "ref_sid_tiny.npz")
VOCAB = 81  # speakers: the dictionary's entries are the classes
SEED = 31
HEAD = "speaker_decoder_postnet."
BASE = dict(mg.TINY, conv_feature_layers=mg.TINY_CONV, feature_grad_mult=1.0, mask_prob=0.0, mask_channel_prob=0.0,
            conv_pos=16, conv_pos_groups=4, max_speech_positions=4000, sid_embed_dim=16)
CASES = {
    "recipe": dict(sid_no_pooling_bn=True, sid_no_embed_postnet=True, sid_pooling_layer="decoder"),
    "defaults": dict(sid_pooling_layer="encoder"),
    "aam": dict(sid_no_pooling_bn=True, sid_no_embed_postnet=True, sid_softmax_type="aamsoftmax", softmax_margin=0.2,
                softmax_scale=30.0),
    "am": dict(sid_no_pooling_bn=True, sid_no_embed_postnet=True, sid_softmax_type="amsoftmax", softmax_margin=0.2,
               softmax_scale=30.0),
}
GRADS = ("speaker_decoder_postnet.output_projection.weight", "speaker_decoder_postnet.output_embedding.weight",
         "speaker_decoder_postnet.bn_embedding.weight", "speaker_decoder_postnet.bn_pooling.weight",
         "decoder.layers.0.encoder_attn.k_proj.weight", "decoder.layers.1.fc2.bias",
         "encoder.layers.0.self_attn.v_proj.weight", "encoder.layers.1.fc1.bias",
         "speech_encoder_prenet.post_extract_proj.weight",
         "speech_encoder_prenet.feature_extractor.conv_layers.0.0.weight")


def batch():
    return synthetic_sid_batch(4, 4000, VOCAB, seed=11)


def case(name, base):
    ns = rl.load()
    args = rl.reference_args(t5_task="s2c", **BASE, **CASES[name])
    torch.manual_seed(777)
    task = rl.RefTask(VOCAB, "s2c")
    model = rl.build_reference_model(args, task).train()
    seed_parameters(model, SEED)
    sample = dict(base, target=base["target"].clone())
    ni = dict(base["net_input"])
    with torch.no_grad():  # row 1 is classified right; with a margin, row 0's target cosine is -1 (< th)
        logits, embed = model(**ni)[0]
        sample["target"][1, 0] = int(logits[1].argmax())
        if name in ("aam", "am"):
            model.speaker_decoder_postnet.output_projection.weight[int(sample["target"][0, 0])] = -embed[0]
    if name in ("aam", "am"):
        ni["target_list"] = sample["target"]
    sample["net_input"] = ni
    seen = {}
    hook = model.speaker_decoder_postnet.register_forward_pre_hook(lambda m, a: seen.__setitem__("x", a[0].detach()))
    cfg = Namespace(post_process="letter", wer_args=None, wer_kenlm_model=None, zero_infinity=False)
    crit = ns.asr_loss.SpeechtoTextLoss(cfg, task, sentence_avg=True, label_smoothing=0.1, report_accuracy=True)
    out = {}
    orig = model.speaker_decoder_postnet.forward

    def keep(*a, **k):
        r = orig(*a, **k)
        out["logits"], out["embed"] = r
        return r
    model.speaker_decoder_postnet.forward = keep
    loss, sample_size, log = crit(model, sample)
    loss.backward()
    model.speaker_decoder_postnet.forward = orig
    hook.remove()
    state = mg._state(model, skip=("text_encoder_prenet.", "speech_decoder_prenet.", "speech_decoder_postnet.",
                                   "text_decoder_postnet."))
    blob = {f"{name}/head/" + k[len("state/" + HEAD):]: v for k, v in state.items() if k.startswith("state/" + HEAD)}
    blob[f"{name}/keys"] = np.array(json.dumps({k[len("state/"):]: list(v.shape) for k, v in state.items()},
                                               sort_keys=True))
    blob[f"{name}/sample/target"] = sample["target"].numpy()
    blob[f"{name}/out/head_input"] = seen["x"].numpy()
    blob[f"{name}/out/logits"] = out["logits"].detach().numpy()
    blob[f"{name}/out/embed"] = out["embed"].detach().numpy()
    blob[f"{name}/loss"] = np.array([log["loss"], log["nll_loss"], log["n_correct"], log["total"], sample_size,
                                     log["ntokens"]], dtype=np.float64)
    named = dict(model.named_parameters())
    for n in GRADS:
        if n in named and named[n].grad is not None:
            blob[f"{name}/grad/" + n] = named[n].grad.numpy()
    model.eval()
    with torch.no_grad():
        pred = model.generate_class(source=ni["source"], prev_output_tokens=ni["prev_output_tokens"],
                                    padding_mask=ni["padding_mask"])
    blob[f"{name}/out/pred"] = pred.numpy()
    return blob


def main():
    base = batch()
    blob = {"batch/in/" + k: base["net_input"][k].numpy() for k in ("source", "padding_mask", "prev_output_tokens")}
    for name in CASES:
        blob.update(case(name, base))
    np.savez_compressed(OUT, **blob)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
