"""Voice conversion (s2s) without a GPU: the reference's own s2s update and synthesis (tests/golden/ref_vc_tiny.npz,
tests/golden/make_golden_vc.py) against the oracle composition (oracle/vc_oracle.py) and against the product model on
emulated kernels; the s2s collater, batch bucketing and host mask draws; the build-time contract."""
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import sid_emulator
from helpers import NO_DROPOUT, TINY, rel

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_vc as mv  # noqa: E402
from oracle import ref_loader as rl  # noqa: E402

needs_ref = pytest.mark.skipif(not rl.available(), reason="reference tree not available")
TRUNK = dict(TINY, **NO_DROPOUT, bert_init=True, build_speech_encoder=True,
             conv_feature_layers="[(32, 10, 5)] + [(32, 3, 2)] * 4 + [(32, 2, 2)] * 2", feature_grad_mult=1.0,
             conv_pos=16, conv_pos_groups=4, use_conv_pos=True, use_sinc_pos=True, mask_prob=0.0, mask_channel_prob=0.0,
             max_speech_positions=4000)


def fixture():
    return dict(np.load(os.path.join(HERE, "golden", "ref_vc_tiny.npz")))


def vc_args(**extra):
    from speecht5_b200.models import make_args
    return make_args("t5_transformer_base_asr", t5_task="s2s", **dict(TRUNK, **extra))


def vc_sample(blob, dev):
    t = lambda k: torch.from_numpy(blob[k]).to(dev)  # noqa: E731
    ni = {k: t("batch/in/" + k) for k in ("source", "padding_mask", "prev_output_tokens", "tgt_lengths", "spkembs")}
    ni["task_name"] = "s2s"
    src_lengths = t("batch/src_lengths")
    return {"id": torch.arange(3), "net_input": ni, "labels": t("batch/labels"), "dec_target": t("batch/dec_target"),
            "dec_target_lengths": t("batch/dec_target_lengths"), "src_lengths": src_lengths, "task_name": "s2s",
            "ntokens": int(blob["batch/src_lengths"].sum()), "target": t("batch/dec_target")}


def vc_case(dev, blob=None):
    """Product model with the reference run's weights (filled from the parameter names) + criterion + batch on `dev`."""
    from speecht5_b200.criterions import SpeechT5Criterion
    from speecht5_b200.tasks import SpeechT5Task
    from test_ref_pin_cpu import seed_parameters
    blob = fixture() if blob is None else blob
    args = vc_args()
    task = SpeechT5Task(args)
    model = task.build_model(args).train()
    seed_parameters(model, mv.SEED)
    model = model.to(dev)
    crit = SpeechT5Criterion(task, use_guided_attn_loss=True)
    return blob, model, crit, vc_sample(blob, dev)


def load_generation_state(model, blob):
    """The post-net BatchNorm statistics the reference's update left."""
    bn = {k[3:]: torch.from_numpy(v) for k, v in blob.items() if k.startswith("bn/")}
    res = model.load_state_dict(bn, strict=False)
    assert not res.unexpected_keys


def generate_cases(model, blob, dev, **extra):
    """generate_speech on the fixture's utterance for every case of make_golden_vc.GEN, each with its stop-logit
    offset: {case: (mel, probs, attn)}."""
    out = {}
    bias = model.speech_decoder_postnet.prob_out.bias
    for name, (kw, offset) in mv.GEN.items():
        with torch.no_grad():
            bias.add_(offset)
        out[name] = model.generate_speech(**gen_inputs(blob, dev), **kw, **extra)
        with torch.no_grad():
            bias.sub_(offset)
    return out


def gen_inputs(blob, dev):
    n = mv.SOURCE_SAMPLES[0]
    t = lambda k: torch.from_numpy(blob["batch/in/" + k]).to(dev)  # noqa: E731
    return dict(source=t("source")[:1, :n], padding_mask=t("padding_mask")[:1, :n], spkembs=t("spkembs")[:1])


# ---------------------------------------------------------------------------------------------- reference pins
@needs_ref
def test_committed_fixture_is_what_the_reference_produces_now():
    fresh = mv.main(path=None)
    stored = fixture()
    assert set(fresh) == set(stored)
    for k in fresh:
        a, b = np.asarray(fresh[k]), stored[k]
        if a.dtype.kind in "biu":
            assert np.array_equal(a, b), k
        else:
            np.testing.assert_allclose(a, b, rtol=1e-5, atol=1e-6, err_msg=k)


@needs_ref
def test_collate_vc_equals_the_reference_collater():
    """speecht5_b200.data.collate_vc against SpeechToSpeechDataset.collater itself (the class compiled from the
    reference source, without its file-reading constructor) on the fixture's items, r = 2 and r = 1."""
    import torch.nn.functional as F
    from speecht5_b200.data import collate_vc
    path = os.path.join(rl.ST5, "speecht5", "data", "speech_to_speech_dataset.py")
    ns = rl._extract(path, ["_collate_frames", "SpeechToSpeechDataset"],
                     {"torch": torch, "np": np, "F": F, "FairseqDataset": object, "List": __import__("typing").List,
                      "Optional": __import__("typing").Optional,
                      "Any": object}, "speecht5.data.speech_to_speech_dataset")
    for r in (2, 1):
        ds = object.__new__(ns["SpeechToSpeechDataset"])
        ds.reduction_factor = r
        items = mv.items()
        want, got = ds.collater(items), collate_vc(items, r)
        assert set(want) == set(got) and set(want["net_input"]) == set(got["net_input"])
        for d_want, d_got in ((want, got), (want["net_input"], got["net_input"])):
            for k, v in d_want.items():
                if torch.is_tensor(v):
                    assert v.dtype == d_got[k].dtype and torch.equal(v, d_got[k]), k
                elif k != "net_input":
                    assert v == d_got[k], k


def _oracle(blob):
    from oracle.speecht5_oracle_asr import base_asr_args, reference_to_oracle_keys
    from oracle.vc_oracle import T5TransformerModelVCOracle
    from speecht5_b200.models import T5TransformerModel
    from test_ref_pin_cpu import seed_parameters
    over = dict(TINY, **NO_DROPOUT, bert_init=True, conv_feature_layers=eval(TRUNK["conv_feature_layers"]),
                feature_grad_mult=1.0, conv_pos=16, conv_pos_groups=4)
    oracle = T5TransformerModelVCOracle(base_asr_args(**over)).train()
    named = T5TransformerModel.build_model(vc_args())
    seed_parameters(named, mv.SEED)
    res = oracle.load_state_dict(reference_to_oracle_keys(named.state_dict()), strict=False)
    assert all(k.endswith(("running_mean", "running_var", "num_batches_tracked")) for k in res.missing_keys), res
    return oracle


def test_oracle_composition_reproduces_the_reference_run():
    """oracle/vc_oracle.py on the fixture's batch: every loss term to 1e-6; outputs and the synthesis from speech (at the
    defaults and with `threshold` passed) to 2e-6 (the post-net output of the reference's own fp32 run is 1.3e-6 from
    the same composition in fp64), the stored gradients to 1e-5."""
    from oracle.vc_oracle import vc_loss
    blob = fixture()
    oracle = _oracle(blob)
    sample = vc_sample(blob, torch.device("cpu"))
    out = oracle(**sample["net_input"])
    for i, k in enumerate(("before", "after", "logits")):
        assert rel(out[i], torch.from_numpy(blob["out/" + k])) < 2e-6, k
    assert rel(torch.stack(out[3]), torch.from_numpy(blob["out/attn"])) < 2e-6
    loss, l1, l2, bce, ga = vc_loss(oracle, out, sample)
    np.testing.assert_allclose([t.item() for t in (loss, l1, l2, bce, ga)], blob["loss"][:5], rtol=1e-6)
    loss.backward()
    from oracle.speecht5_oracle_asr import reference_to_oracle_keys
    named = dict(oracle.named_parameters())
    for k, v in reference_to_oracle_keys({k[5:]: v for k, v in blob.items() if k.startswith("grad/")}).items():
        assert rel(named[k].grad, torch.from_numpy(v)) < 1e-5, k
    oracle.eval()
    load_generation_state(oracle, blob)
    for name, got in generate_cases(oracle, blob, torch.device("cpu")).items():
        for g, k in zip(got, ("mel", "probs", "attn")):
            want = torch.from_numpy(blob[f"gen/{name}/{k}"])
            assert g.shape == want.shape and rel(g, want) < 2e-6, (name, k)


def _batch_norm_act(x, bn, training, act=None, drop_p=0.0):
    """ops.batch_norm_act (the post-net's BatchNorm + tanh) as a differentiable torch call with running statistics."""
    assert drop_p == 0.0 and act in (None, "tanh")
    if training and bn.num_batches_tracked is not None:
        bn.num_batches_tracked += 1
    y = torch.nn.functional.batch_norm(x.float().reshape(-1, x.shape[-1]), bn.running_mean, bn.running_var, bn.weight,
                                       bn.bias, training, bn.momentum, bn.eps)
    y = torch.tanh(y) if act == "tanh" else y
    return y.reshape(x.shape).to(x.dtype)


def _emulated(monkeypatch):
    from speecht5_b200 import ops
    from speecht5_b200.ops import RT
    sid_emulator.install(monkeypatch)
    monkeypatch.setattr(ops, "batch_norm_act", _batch_norm_act)
    monkeypatch.setattr(RT, "dtype", torch.float32)
    RT.clear_static()
    RT.invalidate_shadows()
    return RT


def test_product_update_reproduces_the_reference_run_on_emulated_kernels(monkeypatch):
    """The whole s2s update through the `speecht5` criterion with every kernel emulated (parity arithmetic): loss, every
    logging value and every stored gradient within 2e-4."""
    RT = _emulated(monkeypatch)
    blob, model, crit, sample = vc_case(torch.device("cpu"))
    loss, n, log = crit(model, sample)
    assert n == int(blob["loss"][5])
    assert abs(loss.item() - blob["loss"][0]) < 2e-4 * abs(blob["loss"][0]), (loss.item(), blob["loss"])
    keys = [k[4:] for k in blob if k.startswith("log/")]
    assert set(keys) == set(k for k in log if k != "_stats") and len(keys) >= 10
    for k in keys:
        want = float(blob["log/" + k])
        assert abs(float(log[k]) - want) <= 2e-4 * max(1.0, abs(want)), (k, log[k], want)
    loss.backward()
    params = dict(model.named_parameters())
    grads = [k[5:] for k in blob if k.startswith("grad/")]
    assert len(grads) == len(mv.GRADS)
    for k in grads:
        err = rel(params[k].grad, torch.from_numpy(blob["grad/" + k]))
        assert err < 2e-4, (k, err)
    RT.clear_static()
    RT.invalidate_shadows()


def test_waveform_lengths_as_guided_lengths_miss_the_reference(monkeypatch):
    """The guided-attention loss of an s2s batch needs the conv-frame lengths: fed the raw sample counts (which the
    kernel clips to the encoder length, so every padded frame would count as valid) it misses the reference's value."""
    from speecht5_b200 import frontend
    RT = _emulated(monkeypatch)
    monkeypatch.setattr(frontend.SpeechEncoderPrenet, "get_src_lengths", lambda self, n: n)
    blob, model, crit, sample = vc_case(torch.device("cpu"))
    _, _, log = crit(model, sample)
    want = float(blob["log/enc_dec_attn_loss"])
    assert abs(log["enc_dec_attn_loss"] - want) > 0.05 * want, (log["enc_dec_attn_loss"], want)
    RT.clear_static()
    RT.invalidate_shadows()


@pytest.mark.parametrize("mode", [False, True, "graph_body_eager"])
def test_generate_speech_from_a_waveform_reproduces_the_reference(monkeypatch, mode):
    """generate_speech(source=...) in the prefix, key/value-cache and graph-body modes: mel, stop probabilities and
    cross-attention of the reference's own run: the whole default budget (maxlenratio 10), a stop on a probability
    before it, and `threshold` passed (which also sets minlenratio and maxlenratio)."""
    RT = _emulated(monkeypatch)
    blob, model, _, _ = vc_case(torch.device("cpu"))
    model.eval()
    load_generation_state(model, blob)
    for name, got in generate_cases(model, blob, torch.device("cpu"), use_cache=mode).items():
        for g, k in zip(got, ("mel", "probs", "attn")):
            want = torch.from_numpy(blob[f"gen/{name}/{k}"])
            assert g.shape == want.shape, (name, k, g.shape, want.shape)
            assert rel(g, want) < 1e-4, (name, k, rel(g, want))
    RT.clear_static()
    RT.invalidate_shadows()


def test_task_generate_speech_takes_the_s2s_net_input(monkeypatch):
    """scripts/generate_speech.py hands the task the collated net_input (source, padding_mask, prev_output_tokens,
    tgt_lengths, spkembs, task_name) of a batch of one."""
    from speecht5_b200.data import collate_vc
    from speecht5_b200.tasks import SpeechT5Task
    RT = _emulated(monkeypatch)
    blob, model, _, _ = vc_case(torch.device("cpu"))
    model.eval()
    load_generation_state(model, blob)
    ni = collate_vc(mv.items()[:1])["net_input"]
    with torch.no_grad():
        model.speech_decoder_postnet.prob_out.bias.add_(mv.GEN["default"][1])
    mel, probs, attn = SpeechT5Task(vc_args()).generate_speech([model], ni)
    assert rel(mel, torch.from_numpy(blob["gen/default/mel"])) < 1e-4
    RT.clear_static()
    RT.invalidate_shadows()


# ---------------------------------------------------------------------------------------------- plumbing
def test_synthetic_batch_follows_the_s2s_collater():
    from speecht5_b200.data import synthetic_vc_batch
    s = synthetic_vc_batch(3, 1000, 21, seed=1)
    ni = s["net_input"]
    assert s["task_name"] == ni["task_name"] == "s2s"
    assert s["ntokens"] == int(s["src_lengths"].sum()) and int(s["src_lengths"][0]) == 1000
    assert ni["padding_mask"].shape == ni["source"].shape and not ni["padding_mask"][0].any()
    assert tuple(s["dec_target"].shape) == (3, 21, 80) and int(s["dec_target_lengths"][0]) == 21
    assert tuple(ni["prev_output_tokens"].shape) == (3, 10, 80) and (ni["prev_output_tokens"][:, 0] == 0).all()
    assert torch.equal(ni["prev_output_tokens"][:, 1:], s["dec_target"][:, 1:-2:2])
    assert torch.equal(ni["tgt_lengths"], s["dec_target_lengths"] // 2) and tuple(ni["spkembs"].shape) == (3, 512)


def test_pad_to_buckets_pads_the_waveform_and_the_frames_of_an_s2s_batch():
    from speecht5_b200.data import synthetic_vc_batch
    from speecht5_b200.trainer import pad_to_buckets
    s = synthetic_vc_batch(3, 1000, 21, seed=2)
    p = pad_to_buckets(s, {"wave": 320, "frames": 8, "text": 32, "target": 16})
    ni, pi = s["net_input"], p["net_input"]
    assert pi["source"].shape == (3, 1280) and pi["padding_mask"].shape == (3, 1280)
    assert torch.equal(pi["source"][:, :1000], ni["source"]) and (pi["source"][:, 1000:] == 0).all()
    assert torch.equal(pi["padding_mask"][:, :1000], ni["padding_mask"]) and pi["padding_mask"][:, 1000:].all()
    assert p["dec_target"].shape == (3, 24, 80) and p["labels"].shape == (3, 24) and p["target"].shape == (3, 24, 80)
    assert pi["prev_output_tokens"].shape == (3, 12, 80)
    assert torch.equal(p["dec_target"][:, :21], s["dec_target"]) and torch.equal(p["labels"][:, :21], s["labels"])
    for k in ("dec_target_lengths", "src_lengths"):
        assert torch.equal(p[k], s[k])
    assert torch.equal(pi["tgt_lengths"], ni["tgt_lengths"]) and torch.equal(pi["spkembs"], ni["spkembs"])


def test_host_mask_draws_cover_s2s_batches():
    """With mask_prob / mask_channel_prob > 0 the trainer draws the HuBERT-style masks of an s2s batch on the host (the
    same numpy stream and order as the prenet would) and passes them to forward, so a captured step does not bake one
    draw in."""
    from speecht5_b200.data import draw_hubert_masks, synthetic_vc_batch
    from speecht5_b200.frontend import downsample_padding_mask
    from speecht5_b200.tasks import SpeechT5Task
    from speecht5_b200.trainer import B200Trainer
    args = vc_args(mask_prob=0.5, hubert_mask_length=2, mask_channel_prob=0.25, mask_channel_length=8)
    model = SpeechT5Task(args).build_model(args).train()
    s = synthetic_vc_batch(3, 4000, 20, seed=4)
    fake = SimpleNamespace(model=model, device=torch.device("cpu"), _frame_pm_cache={})
    np.random.seed(9)
    out = B200Trainer._with_host_draws(fake, s)
    pre = model.speech_encoder_prenet
    T = int(pre.get_src_lengths(torch.tensor([4000]))[0])
    np.random.seed(9)
    mi, mc = draw_hubert_masks(pre, 3, T, downsample_padding_mask(s["net_input"]["padding_mask"], T))
    assert torch.equal(out["net_input"]["mask_indices"], mi) and mi.any()
    assert torch.equal(out["net_input"]["mask_channel_indices"], mc) and mc.any()
    model.eval()
    assert B200Trainer._with_host_draws(fake, s) is s  # (no draw outside training)


@pytest.mark.parametrize("extra", [dict(se_predict="masking"), dict(se_predict="target"), dict(se_predict="delta"),
                                   dict(se_decoder_input="source")])
def test_speech_enhancement_variants_raise_at_build_time(extra):
    from speecht5_b200.tasks import SpeechT5Task
    args = vc_args(**extra)
    with pytest.raises(NotImplementedError):
        SpeechT5Task(args).build_model(args)


def test_s2s_metrics_use_the_reference_keys():
    """SpeechT5Criterion.reduce_metrics on s2s logs: s2s_loss / l1 / l2 / bce / decoder_alpha / enc_dec_attn_loss
    (speecht5_criterion.py:285-316; no encoder alpha for s2s)."""
    from speecht5_b200.criterions import SpeechT5Criterion
    from speecht5_b200.fairseq_shim import metrics
    log = {"loss": 1.5, "l1_loss": 1.0, "l2_loss": 2.0, "bce_loss": 0.5, "sample_size": 1, "ntokens": 100,
           "nsentences": 4, "enc_dec_attn_loss": 0.01, "encoder_alpha": 1.0, "decoder_alpha": 1.1}
    logged = {}
    orig = metrics.log_scalar
    metrics.log_scalar = lambda key, value, *a, **k: logged.__setitem__(key, value)
    try:
        SpeechT5Criterion.reduce_metrics([{"s2s": log, "sample_size": 1, "loss": 1.5},
                                          {"s2s": dict(log, loss=2.5), "sample_size": 1, "loss": 2.5}])
    finally:
        metrics.log_scalar = orig
    assert {k for k in logged if k.startswith("s2s_")} == {"s2s_loss", "s2s_l1_loss", "s2s_l2_loss", "s2s_bce_loss",
                                                            "s2s_decoder_alpha", "s2s_enc_dec_attn_loss"}
    assert logged["s2s_loss"] == 2.0 and logged["s2s_decoder_alpha"] == pytest.approx(1.1)
