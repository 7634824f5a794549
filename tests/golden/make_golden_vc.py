"""Generator of tests/golden/ref_vc_tiny.npz: the REFERENCE's own voice-conversion update (T5TransformerModel with
t5_task s2s, models/speecht5.py:786-963: waveform -> conv front end -> encoder, x-vector merged in the speech decoder
prenet, speech decoder post-net) under its TexttoSpeechLoss with the guided-attention loss (default heads and sigma;
criterions/text_to_speech_loss.py:115-214, whose s2s branch :198-206 turns the waveform lengths into conv-frame
lengths), plus its eval-mode generate_speech from a waveform (:1188-1249), at the defaults and with `threshold` passed.

Tiny widths, t5_transformer_base_asr structure with relative positions, reduction factor 2, 512-d x-vectors, every
dropout / LayerDrop / HuBERT mask off. Parameters are not stored: both sides fill every parameter from its NAME
(seed_parameters of tests/test_ref_pin_cpu.py, seed SEED). One batch of 3 with ragged sources (12 / 8 / 5 conv frames)
and ragged targets (30 / 22 / 15 frames).

Stored: batch/<key> (the collated batch), loss [loss, l1, l2, bce, enc_dec_attn_loss, sample_size], log/<key>,
out/{before,after,logits,attn}, grad/<param>, bn/<buffer> (the post-net BatchNorm statistics the update left, which
generation reads), gen/<case>/{mel,probs,attn} for the cases in GEN.

usage: python tests/golden/make_golden_vc.py     (needs the reference tree, see oracle/ref_loader.py)"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import make_golden_from_ref as mg  # noqa: E402
from oracle import ref_loader as rl  # noqa: E402
from speecht5_b200.data import collate_vc  # noqa: E402
from test_ref_pin_cpu import seed_parameters  # noqa: E402

OUT = os.path.join(HERE, "ref_vc_tiny.npz")
VOCAB = 81
SEED = 41
BASE = dict(mg.TINY, conv_feature_layers=mg.TINY_CONV, feature_grad_mult=1.0, mask_prob=0.0, mask_channel_prob=0.0,
            conv_pos=16, conv_pos_groups=4, max_speech_positions=4000)
SOURCE_SAMPLES = (4000, 2900, 1800)
TARGET_FRAMES = (30, 22, 15)
# generation only: (kwargs, stop-logit offset). "default" runs the whole budget (maxlen = 12 * 10 / 2 = 60 steps, no
# probability reaches 0.5), "stop" ends on a stop probability at step 25, "threshold" shows the reference's quirk (the
# passed threshold also sets minlenratio and maxlenratio: minlen = maxlen = 5)
GEN = {"default": ({}, -3.0), "stop": ({}, -2.45), "threshold": ({"threshold": 0.9}, -3.0)}
GRADS = ("speech_encoder_prenet.feature_extractor.conv_layers.0.0.weight",
         "speech_encoder_prenet.post_extract_proj.weight",
         "encoder.layers.0.self_attn.q_proj.weight", "encoder.layers.0.fc1.weight",
         "decoder.layers.0.encoder_attn.k_proj.weight", "decoder.layers.1.encoder_attn.v_proj.bias",
         "speech_decoder_prenet.spkembs_layer.0.weight",
         "speech_decoder_postnet.feat_out.weight", "speech_decoder_postnet.prob_out.weight",
         "speech_decoder_postnet.postnet.postnet.0.0.weight")
BN_PREFIX = "speech_decoder_postnet.postnet."


def items():
    g = torch.Generator().manual_seed(13)
    return [{"id": i, "source": torch.randn(n, generator=g) * 0.1, "target": torch.randn(L, 80, generator=g),
             "spkembs": torch.randn(512, generator=g), "audio_name": f"src{i}", "tgt_name": f"tgt{i}"}
            for i, (n, L) in enumerate(zip(SOURCE_SAMPLES, TARGET_FRAMES))]


def build():
    ns = rl.load()
    args = rl.reference_args(t5_task="s2s", **BASE)
    torch.manual_seed(555)
    task = rl.RefTask(VOCAB, "s2s")
    model = rl.build_reference_model(args, task).train()
    seed_parameters(model, SEED)
    return ns, task, model


def main(path=OUT):
    ns, task, model = build()
    sample = collate_vc(items(), 2)
    crit = ns.tts_loss.TexttoSpeechLoss(task, sentence_avg=True, use_guided_attn_loss=True)
    out = {}
    orig = model.forward

    def keep(*a, **k):
        r = orig(*a, **k)
        out["net"] = r
        return r
    model.forward = keep
    np.random.seed(3)
    loss, sample_size, log = crit(model, sample)
    model.forward = orig
    loss.backward()
    ni = sample["net_input"]
    blob = {"batch/in/" + k: ni[k].numpy() for k in ("source", "padding_mask", "prev_output_tokens", "tgt_lengths",
                                                     "spkembs")}
    for k in ("labels", "dec_target", "dec_target_lengths", "src_lengths"):
        blob["batch/" + k] = sample[k].numpy()
    _, l1, l2, bce, ga = crit.compute_loss(model, out["net"], sample)
    blob["loss"] = np.array([loss.item(), l1.item(), l2.item(), bce.item(), ga.item(), sample_size], dtype=np.float64)
    for k, v in log.items():
        if isinstance(v, (int, float)):
            blob["log/" + k] = np.array(float(v), dtype=np.float64)
    before, after, logits, attn = out["net"]
    blob["out/before"], blob["out/after"], blob["out/logits"] = [t.detach().numpy() for t in (before, after, logits)]
    blob["out/attn"] = torch.stack(list(attn)).detach().numpy()
    named = dict(model.named_parameters())
    for n in GRADS:
        blob["grad/" + n] = named[n].grad.numpy()
    for k, v in model.state_dict().items():
        if k.startswith(BN_PREFIX) and ("running_" in k):
            blob["bn/" + k] = v.numpy()
    model.eval()
    with torch.no_grad():
        n0 = SOURCE_SAMPLES[0]
        bias = model.speech_decoder_postnet.prob_out.bias
        for name, (kw, offset) in GEN.items():
            bias.add_(offset)
            mel, probs, att = model.generate_speech(source=ni["source"][:1, :n0], padding_mask=ni["padding_mask"][:1, :n0],
                                                    spkembs=ni["spkembs"][:1], **kw)
            bias.sub_(offset)
            blob[f"gen/{name}/mel"], blob[f"gen/{name}/probs"], blob[f"gen/{name}/attn"] = (
                mel.numpy(), probs.numpy(), att.numpy())
    if path is not None:
        np.savez_compressed(path, **blob)
        print(path, os.path.getsize(path), "bytes")
    return blob


if __name__ == "__main__":
    main()
