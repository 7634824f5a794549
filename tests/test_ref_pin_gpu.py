"""-m gpu: the CUDA path (through the C ABI) against golden vectors produced by the REFERENCE'S OWN CODE
(tests/golden/ref_*.npz, generator tests/golden/make_golden_from_ref.py, which runs /root/reference/SpeechT5/speecht5
unmodified through oracle/ref_loader.py): the reference's weights and inputs go into the product model, its outputs,
criterion terms, gradients and SequenceGenerator token ids are the expectation. fp32 = parity mode (north_star tolerance
1e-3 on mel), bf16 = throughput mode with its own documented bound. J1 (judge-added row): BASELINE config 1 at FULL
depth (12 + 6 layers, one 4 s utterance) against the CPU oracle."""
import os
import sys

import numpy as np
import pytest
import torch

from helpers import NO_DROPOUT, TINY, rel, to_device

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
VOCAB = 81
TINY_CONV = "[(32, 10, 5)] + [(32, 3, 2)] * 4 + [(32, 2, 2)] * 2"
MEL_TOL = 1e-3     # BASELINE.json north_star: mel L2 within 1e-3 relative (parity mode)
BF16_TOL = 5e-2    # throughput mode on these tiny models with sharpened attention (q, k x6): measured 1-3e-2


def load(name):
    return dict(np.load(os.path.join(GOLD, name + ".npz")))


def state_of(blob, prefix="state/"):
    return {k[len(prefix):]: torch.from_numpy(v) for k, v in blob.items() if k.startswith(prefix)}


def _build(dev, dtype, **over):
    from speecht5_b200.models import T5TransformerModel, make_args
    from speecht5_b200.ops import RT
    RT.dtype = dtype
    RT.manual_seed(1)
    RT.disable_device_seed()
    RT.clear_static()
    RT.invalidate_shadows()
    return T5TransformerModel.build_model(make_args("t5_transformer_base_asr", **over)).to(dev)


class _Dict:
    def __init__(self, n):
        self.n = n

    def __len__(self):
        return self.n

    def pad(self):
        return 1

    def eos(self):
        return 2

    def unk(self):
        return 3

    def index(self, sym):
        return {"<ctc_blank>": self.n - 1, "<mask>": self.n - 2}.get(sym, 3)


class _Task:
    """target_dictionary / blank symbol as tasks/speecht5.py:283-297 sets them up (what the criterion reads)."""
    blank_symbol = "<ctc_blank>"

    def __init__(self, n=VOCAB):
        self.dicts = {"text": _Dict(n)}
        self.target_dictionary = self.dicts["text"]


@pytest.mark.parametrize("dtype,tol", [(torch.float32, MEL_TOL), (torch.bfloat16, BF16_TOL)])
@pytest.mark.parametrize("name,pre_ln", [("ref_tts_tiny", False), ("ref_tts_preln_tiny", True)])
def test_tts_forward_loss_gradients_against_reference_vectors(cuda, name, pre_ln, dtype, tol):
    from speecht5_b200.criterions import TexttoSpeechLoss
    blob = load(name)
    over = dict(TINY, **NO_DROPOUT, bert_init=True)
    if pre_ln:
        over.update(layer_norm_first=True, decoder_normalize_before=True)
    model = _build(cuda, dtype, **over).train()
    model.load_state_dict(state_of(blob))
    ni = {k[3:]: torch.from_numpy(v).to(cuda) for k, v in blob.items() if k.startswith("in/")}
    before, after, logits, attn = model(**ni, task_name="t2s")
    assert rel(after, torch.from_numpy(blob["out/after"])) < tol
    assert rel(before, torch.from_numpy(blob["out/before"])) < tol
    assert rel(logits, torch.from_numpy(blob["out/logits"])) < 3 * tol
    assert rel(torch.stack(attn), torch.from_numpy(blob["out/attn"])) < 3 * tol
    sample = {k[7:]: torch.from_numpy(v).to(cuda) for k, v in blob.items() if k.startswith("sample/")}
    loss, l1, l2, bce, ga = TexttoSpeechLoss(None, use_guided_attn_loss=True).compute_loss(
        model, (before, after, logits, attn), sample)
    got = torch.stack([loss, l1, l2, bce, ga]).detach().cpu().double()
    want = torch.from_numpy(blob["loss"])
    assert ((got - want).abs() / want.abs()).max().item() < 3 * tol
    loss.backward()
    params = dict(model.named_parameters())
    errs = {}
    for k, v in blob.items():
        if k.startswith("grad/"):
            if dtype == torch.bfloat16 and k.endswith("alpha"):
                continue  # a scalar that is a sum of cancelling terms: rounding noise dominates it in bf16
            errs[k] = rel(params[k[5:]].grad, torch.from_numpy(v))
    if dtype == torch.float32:  # parity mode: every gradient, tightly
        assert max(errs.values()) < 3e-3, max(errs.items(), key=lambda kv: kv[1])
    else:
        # throughput mode on a 2 + 2 layer, 64-wide model whose attention the fixture sharpens (q, k x6): single small
        # gradients (the first post-net conv behind BatchNorm over 2 utterances, k_proj of a peaked softmax) carry
        # 0.15-0.45 of bf16 noise on EVERY attention path, the exact fp32 row kernels included. Bound the worst one
        # (cosine > 0.8) and the typical one.
        vals = sorted(errs.values())
        assert vals[-1] < 0.6, max(errs.items(), key=lambda kv: kv[1])
        assert vals[len(vals) // 2] < 0.25, errs


def _asr_model(cuda, dtype, blob, large_style=False):
    over = dict(TINY, **NO_DROPOUT, bert_init=True, build_speech_encoder=True, build_text_decoder=True,
                conv_feature_layers=TINY_CONV, feature_grad_mult=1.0, conv_pos=16, conv_pos_groups=4, use_conv_pos=True,
                use_sinc_pos=True, mask_prob=0.5, hubert_mask_length=4, mask_channel_prob=0.25, mask_channel_length=8,
                max_text_positions=600)
    if large_style:  # t5_transformer_large's structure (models/speecht5.py:1402-1425) on the tiny widths
        over.update(extractor_mode="layer_norm", layer_norm_first=True, decoder_normalize_before=True,
                    share_input_output_embed=True)
    model = _build(cuda, dtype, **over)
    missing = model.load_state_dict(state_of(blob))
    other = ("text_encoder_prenet.", "speech_decoder_prenet.", "speech_decoder_postnet.")  # not on the s2t branch, not stored
    assert not [k for k in missing.missing_keys
                if "num_batches_tracked" not in k and "version" not in k and not k.startswith(other)], missing
    return model


@pytest.mark.parametrize("name,dtype,tol", [("ref_asr_tiny", torch.float32, 1e-3), ("ref_asr_tiny", torch.bfloat16, 4e-2),
                                            ("ref_asr_large_style_tiny", torch.float32, 1e-3),
                                            ("ref_asr_large_style_tiny", torch.bfloat16, 6e-2)])
def test_asr_step_against_reference_vectors(cuda, name, dtype, tol):
    """s2t branch with the reference's OWN mask draws: conv front end, prenet (time + channel masks), encoder + CTC
    head, text decoder; SpeechtoTextLoss CE + CTC and gradients down to conv layer 0 -- the reference's numbers. The
    large-style fixture is t5_transformer_large's structure: the "layer_norm" waveform extractor (per-frame LayerNorm
    after every conv), pre-LN encoder / decoder, tied output embedding."""
    from speecht5_b200.criterions import SpeechT5Criterion
    blob = load(name)
    model = _asr_model(cuda, dtype, blob, large_style="large_style" in name).train()
    ni = dict(source=torch.from_numpy(blob["in/source"]).to(cuda),
              padding_mask=torch.from_numpy(blob["in/padding_mask"]).to(cuda),
              prev_output_tokens=torch.from_numpy(blob["in/prev_output_tokens"]).to(cuda), task_name="s2t",
              mask_indices=torch.from_numpy(blob["in/mask_indices"]).to(cuda),
              mask_channel_indices=torch.from_numpy(blob["in/mask_channel_indices"]).to(cuda))
    sample = {"net_input": ni, "target": torch.from_numpy(blob["sample/target"]).to(cuda),
              "target_lengths": torch.from_numpy(blob["sample/target_lengths"]).to(cuda),
              "ntokens": int(blob["sample/target_lengths"].sum()), "task_name": "s2t"}
    (logits, _), enc = model(**ni)
    assert rel(enc["encoder_out"][0], torch.from_numpy(blob["out/encoder_out"])) < tol
    assert rel(enc["encoder_out_for_ctc"][0], torch.from_numpy(blob["out/encoder_out_for_ctc"])) < 2 * tol
    assert torch.equal(enc["encoder_padding_mask"][0].cpu(), torch.from_numpy(blob["out/encoder_padding_mask"]))
    valid = torch.from_numpy(blob["sample/target"]) != 1  # rows of padded target positions are never read (loss masks them)
    assert rel(logits.cpu()[valid], torch.from_numpy(blob["out/logits"])[valid]) < 2 * tol
    crit = SpeechT5Criterion(_Task(), label_smoothing=0.1, ce_weight=0.5, ctc_weight=0.5, zero_infinity=True)
    loss, _, log = crit(model, sample)
    want = blob["loss"]
    assert abs(loss.item() - want[0]) / abs(want[0]) < 2 * tol, (loss.item(), want, log)
    assert abs(log["ce_loss"] - want[1]) / abs(want[1]) < 2 * tol and abs(log["ctc_loss"] - want[2]) / abs(want[2]) < 2 * tol
    loss.backward()
    params = dict(model.named_parameters())
    gtol = 5e-3 if dtype == torch.float32 else 0.3
    n = 0
    for k, v in blob.items():
        if k.startswith("grad/") and k[5:] in params:
            assert params[k[5:]].grad is not None, k
            assert rel(params[k[5:]].grad, torch.from_numpy(v)) < gtol, (k, rel(params[k[5:]].grad, torch.from_numpy(v)))
            n += 1
    assert n >= 8


@pytest.mark.parametrize("use_cache", [False, True, "graph"])
def test_greedy_token_ids_equal_the_reference_sequence_generator(cuda, use_cache):
    """north_star: bit-exact token ids for ASR greedy decode. Expectation = the reference's own
    speecht5/sequence_generator.py (beam 1) on the reference model; product = CUDA path in parity mode: prefix
    recomputation, the eager key/value cache, and one captured CUDA graph per step (incremental.GreedyGraph; run twice:
    the second call replays the graphs the first one captured)."""
    blob = load("ref_asr_tiny")
    model = _asr_model(cuda, torch.float32, blob).eval()
    hyp = model.generate_text_greedy(torch.from_numpy(blob["in/source"]).to(cuda),
                                     torch.from_numpy(blob["in/padding_mask"]).to(cuda), max_len_b=12,
                                     blank=VOCAB - 1, mask_idx=VOCAB - 2, use_cache=use_cache)
    for b, t in enumerate(hyp):
        n = int(blob["out/greedy_lengths"][b])
        assert t.tolist() == blob["out/greedy_tokens"][b, :n].tolist(), (b, t.tolist())
    if use_cache == "graph":
        again = model.generate_text_greedy(torch.from_numpy(blob["in/source"]).to(cuda),
                                           torch.from_numpy(blob["in/padding_mask"]).to(cuda), max_len_b=12,
                                           blank=VOCAB - 1, mask_idx=VOCAB - 2, use_cache="graph")
        assert [t.tolist() for t in again] == [t.tolist() for t in hyp]


def test_greedy_generator_scores_agree_between_the_eager_cached_and_graph_paths(cuda):
    """speecht5_b200/generator.py (the object task.build_generator returns for beam 1): SequenceGenerator-shaped
    hypotheses whose tokens are the fixture's and whose token log-probabilities agree between the three decoding paths
    (the reference generator's own scores: tests/test_z_reference_model_pins_gpu.py)."""
    from types import SimpleNamespace
    from speecht5_b200.generator import GreedyGenerator
    blob = load("ref_asr_tiny")
    model = _asr_model(cuda, torch.float32, blob).eval()
    vocab = SimpleNamespace(pad=lambda: 1, eos=lambda: 2, unk=lambda: 3)
    sample = {"net_input": {"source": torch.from_numpy(blob["in/source"]).to(cuda),
                            "padding_mask": torch.from_numpy(blob["in/padding_mask"]).to(cuda)}}
    scores = []
    for mode in (False, True, "graph"):
        gen = GreedyGenerator([model], vocab, max_len_b=12, blank=VOCAB - 1, mask_idx=VOCAB - 2, use_cache=mode)
        hypos = gen.generate([model], sample)
        for b, h in enumerate(hypos):
            n = int(blob["out/greedy_lengths"][b])
            assert h[0]["tokens"].tolist() == blob["out/greedy_tokens"][b, :n].tolist()
            assert h[0]["positional_scores"].shape == (n,) and bool((h[0]["positional_scores"] <= 0).all())
            assert abs(float(h[0]["score"]) - float(h[0]["positional_scores"].mean())) < 1e-5
        scores.append(torch.cat([h[0]["positional_scores"] for h in hypos]))
    assert rel(scores[1], scores[0]) < 1e-4 and rel(scores[2], scores[0]) < 1e-4


def test_hifigan_against_the_reference_generator(cuda):
    from oracle.audio_oracle import fold_weight_norm
    from speecht5_b200 import vocoder
    from speecht5_b200.ops import RT
    blob = load("ref_hifigan_tiny")
    cfg = dict(model_in_dim=80, upsample_initial_channel=64, upsample_rates=[4, 4, 4],
               upsample_kernel_sizes=[8, 8, 8], resblock_kernel_sizes=[3, 7, 11],
               resblock_dilation_sizes=[[1, 3, 5]] * 3)
    RT.dtype = torch.bfloat16
    sd = fold_weight_norm(state_of(blob))
    sd["mean"], sd["scale"] = torch.zeros(80), torch.ones(80)
    gen = vocoder.HifiGanGenerator(sd, cfg, device=cuda)
    y = gen(torch.from_numpy(blob["in/mel"]).transpose(1, 2).contiguous().to(cuda), normalize_before=False)
    ref = torch.from_numpy(blob["out/wav"]).squeeze(1)
    assert y.shape == ref.shape
    assert rel(y.float(), ref) < 3e-2  # bf16 activations through 4 up-sampling stages


# ------------------------------------------------------------------------------------------------------------------ J1
@pytest.mark.parametrize("dtype,tol", [(torch.float32, MEL_TOL), (torch.bfloat16, 2.5e-2)])
def test_j1_full_depth_base_config1_mel_l2(cuda, dtype, tol):
    """BASELINE.json config 1 at the real depth: SpeechT5-Base 12 + 6 layers, ONE 4 s utterance (64 text tokens, 250 mel
    frames -> T_dec 125), eval mode, teacher forced, prenet dropout 0 (SURVEY 8d): mel L2 of the CUDA path against the
    fp32 CPU path (oracle, pinned to the reference by tests/test_ref_pin_cpu.py). Parity mode must meet the north_star
    1e-3; bf16 mode is checked against its own bound (bf16 operand rounding alone costs 5.5e-3 at this depth, measured on
    the CPU by rounding every GEMM operand of the oracle)."""
    from oracle.speecht5_oracle import T5TransformerModelOracle, base_args, synthetic_tts_batch
    over = dict(NO_DROPOUT, bert_init=True)
    torch.manual_seed(1337)
    oracle = T5TransformerModelOracle(base_args(**over)).eval()
    sample = synthetic_tts_batch(1, 64, 250, seed=1, ragged=False)
    with torch.no_grad():
        ref = oracle(**sample["net_input"])
    model = _build(cuda, dtype, **over).eval()
    model.load_state_dict(oracle.state_dict())
    with torch.no_grad():
        out = model(**to_device(sample, cuda)["net_input"])
    errs = [rel(out[i], ref[i]) for i in range(3)]
    print(f"J1 {dtype}: before {errs[0]:.3e} after {errs[1]:.3e} logits {errs[2]:.3e}")
    assert errs[1] < tol and errs[0] < tol, errs
