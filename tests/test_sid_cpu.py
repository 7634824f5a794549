"""Speaker identification (s2c) without a GPU: the oracle head against the reference's own run
(tests/golden/ref_sid_tiny.npz, tests/golden/make_golden_sid.py), the product model on emulated kernels against the same
run, the build-time contract of the head, and the margin-CE row program against fp64 autograd."""
import json
import os

import numpy as np
import pytest
import torch

import sid_emulator
from helpers import NO_DROPOUT, TINY, rel

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = ("recipe", "defaults", "aam", "am")
HEAD_PREFIX = "speaker_decoder_postnet."
HEAD = {  # the --sid-* / --softmax-* options of each fixture case (make_golden_sid.CASES)
    "recipe": dict(sid_no_pooling_bn=True, sid_no_embed_postnet=True, sid_pooling_layer="decoder"),
    "defaults": dict(sid_pooling_layer="encoder"),
    "aam": dict(sid_no_pooling_bn=True, sid_no_embed_postnet=True, sid_softmax_type="aamsoftmax", softmax_margin=0.2,
                softmax_scale=30.0),
    "am": dict(sid_no_pooling_bn=True, sid_no_embed_postnet=True, sid_softmax_type="amsoftmax", softmax_margin=0.2,
               softmax_scale=30.0),
}
TRUNK = dict(TINY, **NO_DROPOUT, bert_init=True, build_speech_encoder=True, build_text_decoder=True,
             conv_feature_layers="[(32, 10, 5)] + [(32, 3, 2)] * 4 + [(32, 2, 2)] * 2", feature_grad_mult=1.0,
             conv_pos=16, conv_pos_groups=4, use_conv_pos=True, use_sinc_pos=True, mask_prob=0.0, mask_channel_prob=0.0,
             max_speech_positions=4000, sid_embed_dim=16)


def fixture():
    return dict(np.load(os.path.join(HERE, "golden", "ref_sid_tiny.npz")))


def sid_args(name, **extra):
    from speecht5_b200.models import make_args
    return make_args("t5_transformer_base_asr", t5_task="s2c", **dict(TRUNK, **HEAD[name], **extra))


SEED = 31  # make_golden_sid.SEED: every parameter is filled from its name, like the reference model was


def head_state(blob, name):
    """The speaker head's parameters and buffers as the reference run left them (full state-dict names)."""
    pre = f"{name}/head/"
    return {HEAD_PREFIX + k[len(pre):]: torch.from_numpy(v) for k, v in blob.items() if k.startswith(pre)}


def sid_case(name, dev, blob=None):
    """Product model with the reference run's weights + the criterion and batch of case `name` on `dev`."""
    from speecht5_b200.criterions import SpeechT5Criterion
    from speecht5_b200.tasks import SpeechT5Task
    from test_ref_pin_cpu import seed_parameters
    blob = fixture() if blob is None else blob
    args = sid_args(name)
    task = SpeechT5Task(args)
    model = task.build_model(args).train()
    seed_parameters(model, SEED)
    missing = model.load_state_dict(head_state(blob, name), strict=False)
    assert not missing.unexpected_keys and not [k for k in missing.missing_keys if k.startswith(HEAD_PREFIX)], missing
    model = model.to(dev)
    b = lambda k: torch.from_numpy(blob[f"batch/{k}"]).to(dev)  # noqa: E731
    t = lambda k: torch.from_numpy(blob[f"{name}/{k}"]).to(dev)  # noqa: E731
    ni = dict(source=b("in/source"), padding_mask=b("in/padding_mask"), prev_output_tokens=b("in/prev_output_tokens"),
              task_name="s2c")
    if name in ("aam", "am"):
        ni["target_list"] = t("sample/target")
    B = ni["source"].shape[0]
    sample = {"id": torch.arange(B), "task_name": "s2c", "net_input": ni, "target": t("sample/target"),
              "target_lengths": torch.ones(B, dtype=torch.long, device=dev), "ntokens": B}
    crit = SpeechT5Criterion(task, label_smoothing=0.1, report_accuracy=True)
    return blob, model, crit, sample


def _oracle_kw(name):
    h = HEAD[name]
    return dict(softmax_type=h.get("sid_softmax_type", "softmax"), pooling_bn=not h.get("sid_no_pooling_bn", False),
                embed_postnet=not h.get("sid_no_embed_postnet", False), scale=h.get("softmax_scale", 1.0),
                margin_m=h.get("softmax_margin", 0.0))


@pytest.mark.parametrize("name", CASES)
def test_oracle_head_reproduces_the_reference_run(name):
    """oracle/speaker_oracle.py on the head input the reference's head received: its logits, embedding, criterion
    values and head-weight gradient."""
    from oracle.speaker_oracle import label_smoothed_ce, speaker_head
    blob = fixture()
    state = {k: v.double() for k, v in head_state(blob, name).items()}
    w = state["speaker_decoder_postnet.output_projection.weight"].requires_grad_()
    target = torch.from_numpy(blob[f"{name}/sample/target"])[:, 0]
    logits, embed = speaker_head(state, torch.from_numpy(blob[f"{name}/out/head_input"]), target=target,
                                 **_oracle_kw(name))
    np.testing.assert_allclose(logits.detach().numpy(), blob[f"{name}/out/logits"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(embed.detach().numpy(), blob[f"{name}/out/embed"], rtol=1e-6, atol=1e-6)
    loss, nll, correct, total = label_smoothed_ce(logits, target, 0.1)
    want = blob[f"{name}/loss"]
    assert abs(loss.item() - want[0]) <= 1e-6 * abs(want[0]) and abs(nll.item() - want[1]) <= 1e-6 * abs(want[1])
    assert (correct, total) == (int(want[2]), int(want[3]))
    loss.backward()
    assert rel(w.grad, torch.from_numpy(blob[f"{name}/grad/speaker_decoder_postnet.output_projection.weight"])) < 1e-6


@pytest.mark.parametrize("name", CASES)
def test_product_update_reproduces_the_reference_run_on_emulated_kernels(monkeypatch, name):
    """The whole s2c update through the `speecht5` criterion with every kernel emulated (parity arithmetic): loss,
    logging values, sample size, the logits and embedding, and the stored gradients within 2e-4; then the eval-mode
    generate_class predictions."""
    from speecht5_b200.ops import RT
    sid_emulator.install(monkeypatch)
    monkeypatch.setattr(RT, "dtype", torch.float32)
    RT.clear_static()
    RT.invalidate_shadows()
    blob, model, crit, sample = sid_case(name, torch.device("cpu"))
    seen = {}
    model.speaker_decoder_postnet.register_forward_hook(lambda m, a, out: seen.__setitem__("out", out))
    loss, n, log = crit(model, sample)
    want = blob[f"{name}/loss"]
    assert n == int(want[4]) and log["ntokens"] == int(want[5]) and log["sample_size"] == int(want[4])
    assert abs(loss.item() - want[0]) < 2e-4 * abs(want[0]), (loss.item(), want)
    assert abs(log["nll_loss"] - want[1]) < 2e-4 * abs(want[1]) and log["ce_loss"] == log["loss"]
    assert (log["n_correct"], log["total"]) == (int(want[2]), int(want[3]))
    assert rel(seen["out"][0], torch.from_numpy(blob[f"{name}/out/logits"])) < 2e-4
    assert rel(seen["out"][1], torch.from_numpy(blob[f"{name}/out/embed"])) < 2e-4
    loss.backward()
    params = dict(model.named_parameters())
    grads = [k[len(name) + 6:] for k in blob if k.startswith(name + "/grad/")]
    assert len(grads) >= 6
    for k in grads:
        assert params[k].grad is not None, k
        err = rel(params[k].grad, torch.from_numpy(blob[f"{name}/grad/{k}"]))
        assert err < 2e-4, (k, err)
    model.load_state_dict(head_state(blob, name), strict=False)  # BatchNorm statistics of the reference's eval
    model.eval()
    ni = sample["net_input"]
    pred = model.generate_class(ni["source"], ni["prev_output_tokens"], padding_mask=ni["padding_mask"])
    assert pred.tolist() == blob[f"{name}/out/pred"].tolist()
    RT.clear_static()
    RT.invalidate_shadows()


def test_state_dict_keys_and_shapes_equal_the_reference_model():
    """Every head and trunk parameter / buffer the reference's s2c model carries, with its shape (checkpoints load)."""
    from speecht5_b200.models import T5TransformerModel
    blob = fixture()
    from speecht5_b200.tasks import SpeechT5Task
    for name in ("recipe", "defaults"):
        args = sid_args(name)
        model = T5TransformerModel.build_model(args, SpeechT5Task(args))
        ours = {k: tuple(v.shape) for k, v in model.state_dict().items() if "num_batches_tracked" not in k
                and not k.startswith(("text_encoder_prenet.", "speech_decoder_", "text_decoder_postnet."))}
        ref = {k: tuple(v) for k, v in json.loads(str(blob[f"{name}/keys"])).items()}
        assert ours == ref
    assert "speaker_decoder_postnet.bn_pooling.running_var" in ref and "speaker_decoder_postnet.bn_embedding.weight" in ref


@pytest.mark.parametrize("extra", [dict(sid_pooling_layer="decoder-las"), dict(sid_pooling_layer="encoder-cls"),
                                   dict(sid_pooling_layer="encoder-speaker"), dict(sid_t5_postnet=True),
                                   dict(sid_encoder_cls="encoder"), dict(sid_shuffle_encoder_input=True),
                                   dict(sid_decoder_speaker=True), dict(sid_pad_prenet=True),
                                   dict(build_text_decoder=False), dict(build_speech_encoder=False)])
def test_unbuilt_speaker_variants_raise_at_build_time(extra):
    from speecht5_b200.tasks import SpeechT5Task
    args = sid_args("recipe")
    for k, v in extra.items():
        setattr(args, k, v)
    with pytest.raises(NotImplementedError):
        SpeechT5Task(args).build_model(args)


def test_model_without_the_head_keeps_the_vocabulary_path_on_an_s2c_batch(monkeypatch):
    """A speech-in / text-out model built for another task has no speaker head: an s2c batch takes the old path (the
    text decoder and its vocabulary projection), exactly as before the head existed."""
    from speecht5_b200.data import synthetic_sid_batch
    from speecht5_b200.ops import RT
    from speecht5_b200.tasks import SpeechT5Task
    sid_emulator.install(monkeypatch)
    monkeypatch.setattr(RT, "dtype", torch.float32)
    RT.invalidate_shadows()
    args = sid_args("recipe")
    args.t5_task = "s2t"
    model = SpeechT5Task(args).build_model(args).eval()
    assert model.speaker_decoder_postnet is None
    sample = synthetic_sid_batch(2, 4000, 81, seed=3)
    with torch.no_grad():
        out = model(**sample["net_input"])
    assert len(out) == 3 and out[0][1] is None and tuple(out[0][0].shape) == (2, 1, 81)
    RT.invalidate_shadows()


def test_synthetic_batch_follows_the_s2c_collater():
    from speecht5_b200.data import synthetic_sid_batch
    s = synthetic_sid_batch(3, 1000, 40, seed=1)
    ni = s["net_input"]
    assert s["task_name"] == ni["task_name"] == "s2c" and s["ntokens"] == 3
    assert ni["prev_output_tokens"].tolist() == [[2], [2], [2]] and tuple(s["target"].shape) == (3, 1)
    assert ((s["target"] >= 4) & (s["target"] < 38)).all()
    assert ni["padding_mask"].shape == ni["source"].shape and not ni["padding_mask"][0].any()


@pytest.mark.parametrize("kind,easy", [("softmax", False), ("amsoftmax", False), ("aamsoftmax", False),
                                       ("aamsoftmax", True)])
@pytest.mark.parametrize("eps", [0.0, 0.1])
def test_margin_ce_row_program_matches_fp64_autograd(kind, easy, eps):
    """The kernels' row program (tests/sid_emulator.py: closed-form margin logit and slope, smoothing as N lse - sum z,
    gradient from the saved lse) against torch fp64 autograd through the reference's formulas; rows on both sides of
    th = cos(pi - m) and of 0, an ignored row, and a correct row."""
    from oracle.speaker_oracle import label_smoothed_ce, margin
    g = torch.Generator().manual_seed(5)
    B, N, m, s = 6, 37, 0.2, 30.0
    cos = (torch.rand(B, N, generator=g, dtype=torch.float64) * 2 - 1) * 0.9
    target = torch.randint(4, N, (B,), generator=g)
    cos[0, target[0]] = -0.995  # below th
    cos[1, target[1]] = -0.5    # above th, below 0
    cos[2, target[2]] = 0.99    # arg-max
    target[3] = 1               # padding row: ignored
    cos = cos.float().double()
    x = cos.clone().requires_grad_()
    z = x if kind == "softmax" else margin(x, target, kind, m, s, easy)
    loss, nll, correct, total = label_smoothed_ce(z, target, eps, ignore_index=1)
    (1.3 * loss + 0.7 * nll).backward()
    mode = {"softmax": None, "amsoftmax": (sid_emulator.AM, s, m, 0), "aamsoftmax": (sid_emulator.AAM, s, m, int(easy))}[kind]
    mt = None if mode is None else target
    zk = torch.empty(B, N)
    sid_emulator.margin_ce_fwd(cos.float(), mt, mode, z_out=zk)
    stats, lse = torch.empty(B, 4), torch.empty(B)
    sid_emulator.margin_ce_fwd(cos.float(), mt, mode, target=target, eps=eps, ignore_index=1, stats=stats, lse=lse)
    assert rel(zk, z) < 1e-6
    assert abs(stats[:, 0].sum().item() - loss.item()) < 1e-5 * abs(loss.item())
    assert abs(stats[:, 1].sum().item() - nll.item()) < 1e-5 * abs(nll.item())
    assert (int(stats[:, 2].sum()), int(stats[:, 3].sum())) == (correct, total) and total == B - 1
    dx = torch.empty(B, N)
    sid_emulator.margin_ce_bwd(cos.float(), mt, mode, dx, target=target, eps=eps, ignore_index=1, lse=lse,
                               gstat=torch.tensor([1.3, 0.7]))
    assert rel(dx, x.grad) < 1e-5
    # the two halves the model and the criterion issue: margin logits, then plain CE on them
    dz = torch.empty(B, N)
    sid_emulator.margin_ce_fwd(zk, None, None, target=target, eps=eps, ignore_index=1, stats=stats, lse=lse)
    sid_emulator.margin_ce_bwd(zk, None, None, dz, target=target, eps=eps, ignore_index=1, lse=lse,
                               gstat=torch.tensor([1.3, 0.7]))
    sid_emulator.margin_ce_bwd(cos.float(), mt, mode, dx, dz=dz)
    assert rel(dx, x.grad) < 1e-5
