"""-m gpu: the speech-input front end (speecht5_b200/frontend.py + csrc/conv_frontend.cu), CE + CTC criterion, greedy
decoding, KV cache, log-mel, HiFi-GAN and the pre-training extras against the oracles."""
import os

import pytest
import torch

pytestmark = [pytest.mark.gpu]


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


def _args():
    from oracle import speecht5_oracle_asr as O
    args = O.base_asr_args(encoder_layers=1, decoder_layers=1, dropout=0.0)
    for k, v in dict(encoder_speech_prenet="conv", mask_prob=0.0, hubert_mask_length=10, mask_selection="static",
                     mask_other=0.0, no_mask_overlap=False, mask_min_space=1).items():
        setattr(args, k, v)
    args.conv_feature_layers = list(O.CONV_FEATURE_LAYERS)  # a list suits both the oracle and the product
    return args


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_feature_extractor_forward_backward(cuda, dtype):
    from oracle import speecht5_oracle_asr as O
    from speecht5_b200 import frontend
    from speecht5_b200.ops import RT
    RT.dtype = dtype
    RT.invalidate_shadows()
    torch.manual_seed(0)
    ref = O.ConvFeatureExtractionModel().double()
    mine = frontend.ConvFeatureExtractor().to(cuda)
    mine.load_state_dict({k: v.float() for k, v in ref.state_dict().items()})
    wave = torch.randn(2, 9000, dtype=torch.float64) * 0.3
    yr = ref(wave).transpose(1, 2)
    dy = torch.randn_like(yr)
    yr.backward(dy)
    y = mine(wave.float().to(cuda))
    y.backward(dy.to(cuda).to(y.dtype))
    tol = 5e-5 if dtype == torch.float32 else 3e-2
    assert y.shape == yr.shape
    assert rel(y.cpu(), yr) < tol
    gr = dict(ref.named_parameters())
    for n, p in mine.named_parameters():
        assert rel(p.grad.cpu(), gr[n].grad) < tol * 4, n
    RT.dtype = torch.bfloat16


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_speech_encoder_prenet_against_the_oracle(cuda, dtype):
    from oracle import speecht5_oracle_asr as O
    from speecht5_b200 import frontend
    from speecht5_b200.ops import RT
    RT.dtype = dtype
    RT.invalidate_shadows()
    torch.manual_seed(1)
    args = _args()
    ref = O.SpeechEncoderPrenet(args).double().eval()
    mine = frontend.SpeechEncoderPrenet(args).to(cuda).eval()
    sd = {k: v.float() for k, v in ref.state_dict().items()}
    sd["pos_conv.0.weight_g"] = sd.pop("pos_conv_g")
    sd["pos_conv.0.weight_v"] = sd.pop("pos_conv_v")
    sd["pos_conv.0.bias"] = sd.pop("pos_conv_bias")
    missing, unexpected = mine.load_state_dict(sd, strict=False)
    assert not unexpected and not missing, (missing, unexpected)
    B, n = 2, 8000
    wave = torch.randn(B, n, dtype=torch.float64) * 0.3
    lengths = torch.tensor([8000, 5000])
    pm = torch.arange(n)[None, :] >= lengths[:, None]
    T = int(ref.feature_extractor.get_out_seq_lens_tensor(torch.tensor([n]))[0])
    mi = torch.zeros(B, T, dtype=torch.bool)
    mi[0, 3:9] = True
    mi[1, 1:4] = True
    xr, mr, pen_r = ref(wave, pm, mask_indices=mi)
    (x, pen, _, _), m = mine(wave.float().to(cuda), require_feat_pen=True, padding_mask=pm.to(cuda), mask=True,
                             mask_indices=mi.to(cuda))
    tol = 1e-4 if dtype == torch.float32 else 3e-2
    assert torch.equal(m.cpu(), mr)
    assert rel(x.cpu(), xr) < tol
    assert abs(pen.item() - pen_r.item()) / pen_r.item() < tol
    RT.dtype = torch.bfloat16


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_speech_to_text_step_against_the_oracle(cuda, dtype):
    """Opt-in s2t branch end to end (waveform front end -> encoder + CTC head -> text decoder): logits, CE + CTC loss
    and a few gradients vs oracle T5TransformerModelASROracle / asr_loss (SURVEY 8d config 3 shapes, reduced)."""
    from oracle import speecht5_oracle_asr as O
    from speecht5_b200.criterions import SpeechT5Criterion
    from speecht5_b200.models import T5TransformerModel, make_args
    from speecht5_b200.ops import RT
    RT.dtype = dtype
    RT.manual_seed(1)
    RT.invalidate_shadows()
    torch.manual_seed(4)
    over = dict(encoder_layers=2, decoder_layers=2, bert_init=True, dropout=0.0, attention_dropout=0.0,
                activation_dropout=0.0, encoder_layerdrop=0.0, decoder_layerdrop=0.0, mask_prob=0.0,
                mask_channel_prob=0.0, feature_grad_mult=1.0)
    oracle = O.T5TransformerModelASROracle(O.base_asr_args(**over)).train()
    args = make_args("t5_transformer_base_asr", build_speech_encoder=True, build_text_decoder=True, use_conv_pos=True,
                     use_sinc_pos=True, **over)
    model = T5TransformerModel.build_model(args).to(cuda).train()
    sd = dict(oracle.state_dict())
    for a, b in (("pos_conv_g", "pos_conv.0.weight_g"), ("pos_conv_v", "pos_conv.0.weight_v"),
                 ("pos_conv_bias", "pos_conv.0.bias")):
        sd["speech_encoder_prenet." + b] = sd.pop("speech_encoder_prenet." + a)
    model.load_state_dict(sd)
    s = O.synthetic_asr_batch(2, 16000, 12, seed=3)
    want, ce, ctc, _ = O.asr_loss(oracle, s, ce_weight=0.5, ctc_weight=0.5, label_smoothing=0.1)
    want.backward()
    sample = {"net_input": {k: (v.to(cuda) if torch.is_tensor(v) else v) for k, v in s["net_input"].items()},
              "target": s["target"].to(cuda), "target_lengths": s["target_lengths"].to(cuda), "ntokens": s["ntokens"],
              "task_name": "s2t"}
    crit = SpeechT5Criterion(None, label_smoothing=0.1, ce_weight=0.5, ctc_weight=0.5)
    loss, _, log = crit(model, sample)
    tol = 1e-3 if dtype == torch.float32 else 6e-2
    assert abs(loss.item() - want.item()) / abs(want.item()) < tol, (loss.item(), want.item(), log)
    loss.backward()
    ref, got = dict(oracle.named_parameters()), dict(model.named_parameters())
    gtol = 1e-2 if dtype == torch.float32 else 0.3
    for name in ("speech_encoder_prenet.feature_extractor.conv_layers.3.0.weight",
                 "speech_encoder_prenet.feature_extractor.conv_layers.0.0.weight",
                 "speech_encoder_prenet.post_extract_proj.weight", "encoder.layers.1.fc1.weight",
                 "decoder.layers.0.encoder_attn.q_proj.weight", "encoder.proj.weight"):
        assert rel(got[name].grad.cpu(), ref[name].grad) < gtol, name
    wg = got["speech_encoder_prenet.pos_conv.0.weight_v"].grad.cpu()
    assert rel(wg, ref["speech_encoder_prenet.pos_conv_v"].grad) < gtol
    RT.dtype = torch.bfloat16


def test_logmel_on_device_against_the_oracle(cuda):
    """speecht5_b200/audio.py (STFT and mel projection on the wgmma GEMM, split precision) vs oracle/audio_oracle.py."""
    import numpy as np
    from oracle.audio_oracle import logmelfilterbank as ref_fn
    from speecht5_b200 import audio
    rng = np.random.default_rng(3)
    n = 16000 * 2 + 77
    t = np.arange(n) / 16000.0
    waves = np.stack([0.3 * np.sin(2 * np.pi * 300 * t) + 0.02 * rng.standard_normal(n),
                      0.1 * np.sin(2 * np.pi * 2500 * t) + 0.05 * rng.standard_normal(n)]).astype(np.float32)
    got = audio.logmelfilterbank(torch.from_numpy(waves).to(cuda)).cpu().numpy()
    want = np.stack([ref_fn(w) for w in waves])
    assert got.shape == want.shape
    assert np.abs(got - want).max() < 2e-3, np.abs(got - want).max()


def test_greedy_text_decoding_token_ids_match_the_oracle(cuda):
    """SURVEY 8a row 21 (ASR half): beam-1 decoding on the device path (prefix recomputation) gives the oracle's token
    ids (fp32 parity mode; random weights make near-ties unlikely but the logits are also compared)."""
    from oracle import speecht5_oracle_asr as O
    from speecht5_b200.models import T5TransformerModel, make_args
    from speecht5_b200.ops import RT
    RT.dtype = torch.float32
    RT.invalidate_shadows()
    torch.manual_seed(6)
    over = dict(encoder_layers=2, decoder_layers=2, bert_init=True, mask_prob=0.0, mask_channel_prob=0.0)
    oracle = O.T5TransformerModelASROracle(O.base_asr_args(**over)).eval()
    with torch.no_grad():
        oracle.text_decoder_postnet.output_projection.weight.mul_(8.0)  # spread the logits
    args = make_args("t5_transformer_base_asr", build_speech_encoder=True, build_text_decoder=True, use_conv_pos=True,
                     use_sinc_pos=True, **over)
    model = T5TransformerModel.build_model(args).to(cuda).eval()
    sd = dict(oracle.state_dict())
    for a, b in (("pos_conv_g", "pos_conv.0.weight_g"), ("pos_conv_v", "pos_conv.0.weight_v"),
                 ("pos_conv_bias", "pos_conv.0.bias")):
        sd["speech_encoder_prenet." + b] = sd.pop("speech_encoder_prenet." + a)
    model.load_state_dict(sd)
    s = O.synthetic_asr_batch(2, 12000, 6, seed=9)
    src, pm = s["net_input"]["source"], s["net_input"]["padding_mask"]
    want = O.greedy_decode(oracle, src, pm, max_len_b=12)
    got = model.generate_text_greedy(src.to(cuda), pm.to(cuda), max_len_b=12)
    assert [t.tolist() for t in got] == [t.tolist() for t in want]
    RT.dtype = torch.bfloat16


def test_ctc_kernel_against_torch(cuda):
    """csrc/ctc.cu (fused log-softmax + CTC nll + logit gradient) vs torch's ctc_loss autograd: ASR-shaped batch with
    ragged input / target lengths, repeated labels and one infeasible utterance under zero_infinity."""
    import torch.nn.functional as F
    from speecht5_b200.frontend import ctc_loss_sum
    torch.manual_seed(13)
    T, B, V = 120, 5, 81
    tl = torch.tensor([30, 12, 1, 70, 25])
    il = torch.tensor([120, 90, 3, 100, 120])  # utterance 3: 70 labels in 100 frames is feasible only without repeats
    tg = [torch.randint(1, V, (int(n),)) for n in tl]
    tg[3][::2] = tg[3][1::2]  # repeated pairs -> needs 70 + 35 = 105 frames > 100: infeasible
    flat = torch.cat(tg)
    logits = torch.randn(T, B, V, requires_grad=True)
    ref = F.ctc_loss(F.log_softmax(logits, -1), flat, il, tl, blank=0, reduction="sum", zero_infinity=True)
    ref.backward()
    x = logits.detach().to(cuda).requires_grad_()
    got = ctc_loss_sum(x, flat.to(cuda), il.to(cuda), tl.to(cuda), 0, True)
    (got * 2.0).backward()
    assert abs(got.item() - ref.item()) < 1e-4 * abs(ref.item())
    assert rel(x.grad.cpu() / 2.0, logits.grad) < 1e-4
    assert x.grad[:, 3].abs().max().item() == 0.0 and x.grad[100:, 1].abs().max().item() == 0.0


@pytest.mark.parametrize("T,B,V,lens", [(499, 8, 81, (160, 150, 97, 160, 3, 120, 160, 33)),   # the ASR step: S = 321
                                           (700, 3, 40, (300, 10, 257))])                        # S = 601: sweeps one after the other
def test_ctc_kernel_long_sequences_against_torch(cuda, T, B, V, lens):
    """csrc/ctc.cu at the benched ASR shape (alpha / beta recursions side by side in one CTA) and beyond 512 states (the
    same kernel runs the two recursions one after the other), ragged lengths, vs torch's ctc_loss autograd; also through
    the padded-target entry the captured step uses."""
    import torch.nn.functional as F
    from speecht5_b200.frontend import ctc_loss_sum, ctc_loss_sum_padded
    torch.manual_seed(5)
    tl = torch.tensor(lens)
    il = torch.tensor([T - 7 * (i % 3) for i in range(B)])
    tg = [torch.randint(1, V, (int(n),)) for n in tl]
    tg[1][1::3] = tg[1][0::3][:len(tg[1][1::3])]  # some repeated labels
    flat = torch.cat(tg)
    # fp64 reference: an fp32 log-domain lattice holds values of magnitude T * log V ~ 2000, i.e. 1 ulp = 1e-4 .. 2.5e-4
    # absolute = the relative error of every posterior term; torch's own fp32 path is measured next to ours
    logits = (torch.randn(T, B, V) * 2).double().requires_grad_()
    ref = F.ctc_loss(F.log_softmax(logits, -1), flat, il, tl, blank=0, reduction="sum", zero_infinity=True)
    ref.backward()
    l32 = logits.detach().float().requires_grad_()
    F.ctc_loss(F.log_softmax(l32, -1), flat, il, tl, blank=0, reduction="sum", zero_infinity=True).backward()
    torch_fp32_err = rel(l32.grad, logits.grad)
    x = logits.detach().float().to(cuda).requires_grad_()
    got = ctc_loss_sum(x, flat.to(cuda), il.to(cuda), tl.to(cuda), 0, True)
    got.backward()
    assert abs(got.item() - ref.item()) < 1e-4 * abs(ref.item())
    assert rel(x.grad.cpu(), logits.grad) < max(2e-3, 4 * torch_fp32_err), (rel(x.grad.cpu(), logits.grad), torch_fp32_err)
    padded = torch.zeros(B, int(tl.max()), dtype=torch.long)
    for i, t_ in enumerate(tg):
        padded[i, :len(t_)] = t_
    x2 = logits.detach().float().to(cuda).requires_grad_()
    got2 = ctc_loss_sum_padded(x2, padded.to(cuda), il.to(cuda), tl.to(cuda), 0, True)
    got2.backward()
    assert abs(got2.item() - ref.item()) < 1e-4 * abs(ref.item()) and rel(x2.grad, x.grad) < 1e-5


def test_hifigan_on_device_against_the_oracle(cuda):
    """speecht5_b200/vocoder.py with the release configuration (512 channels, 4x4x4x4 up-sampling, ResBlocks 3/7/11 x
    dilations 1/3/5) vs oracle HifiGanGenerator (fp32 CPU) on a short mel: bf16 activations, so a relative L2 bound."""
    from oracle.audio_oracle import HifiGanGenerator as Ref
    from speecht5_b200 import vocoder
    torch.manual_seed(0)
    ref = Ref(std=0.02, seed=1).eval()
    gen = vocoder.HifiGanGenerator(ref.state_dict(), device=cuda)
    mel = torch.randn(2, 37, 80)
    with torch.no_grad():
        want = ref(mel)
    got = gen(mel.to(cuda)).cpu()
    assert got.shape == want.shape == (2, 37 * 256)
    assert rel(got, want) < 3e-2


def test_kv_cache_synthesis_equals_prefix_recomputation(cuda):
    """speecht5_b200/incremental.py on the device: greedy speech synthesis with the key/value cache (one-row attention
    on the row kernels over strided cache views) vs the validated prefix-recomputing path (fp32 parity mode, prenet
    dropout off so both runs see the same numbers)."""
    from helpers import NO_DROPOUT
    from speecht5_b200.models import T5TransformerModel, make_args
    from speecht5_b200.ops import RT
    RT.dtype = torch.float32
    RT.invalidate_shadows()
    torch.manual_seed(3)
    over = dict(encoder_layers=2, decoder_layers=2, bert_init=True, **NO_DROPOUT)
    tts = T5TransformerModel.build_model(make_args("t5_transformer_base_asr", **over)).to(cuda).eval()
    with torch.no_grad():
        tts.speech_decoder_postnet.prob_out.bias.fill_(-2.0)
    tok = torch.randint(4, 81, (1, 23), device=cuda)
    spk = torch.randn(1, 512, device=cuda)
    plain = tts.generate_speech(src_tokens=tok, spkembs=spk, threshold=0.9)
    cached = tts.generate_speech(src_tokens=tok, spkembs=spk, threshold=0.9, use_cache=True)
    graphed = tts.generate_speech(src_tokens=tok, spkembs=spk, threshold=0.9, use_cache="graph")  # one replay per step
    for a, b, c in zip(plain, cached, graphed):
        assert a.shape == b.shape == c.shape and rel(b, a) < 1e-4 and rel(c, b) < 1e-5
    RT.dtype = torch.bfloat16


def test_graph_captured_synthesis_in_throughput_mode(cuda):
    """SynthesisGraph (speecht5_b200/incremental.py) in bf16 with the always-on prenet dropout: more steps than one span
    bucket (two graphs), a new dropout mask per replay from the device-resident seed (steps with identical inputs give
    different frames), and the same seed gives the same utterance again."""
    from speecht5_b200.models import T5TransformerModel, make_args
    from speecht5_b200.ops import RT
    RT.dtype = torch.bfloat16
    RT.invalidate_shadows()
    torch.manual_seed(5)
    tts = T5TransformerModel.build_model(make_args("t5_transformer_base_asr", encoder_layers=2, decoder_layers=2,
                                                   bert_init=True)).to(cuda).eval()
    tok = torch.randint(4, 81, (1, 150), device=cuda)
    spk = torch.randn(1, 512, device=cuda)
    runs = []
    for _ in range(2):
        RT.manual_seed(7)
        runs.append(tts.generate_speech(src_tokens=tok, spkembs=spk, threshold=2.0, use_cache="graph"))  # maxlen = 150 steps
    mel, probs, attn = runs[0]
    assert mel.shape == (300, 80) and probs.shape == (300,) and attn.shape == (2, 12, 150, 150)
    assert torch.isfinite(mel).all() and torch.isfinite(attn).all()
    assert (attn.sum(-1) - 1).abs().max() < 1e-3
    for a, b in zip(runs[0], runs[1]):
        assert torch.equal(a, b)
    RT.manual_seed(8)
    other = tts.generate_speech(src_tokens=tok, spkembs=spk, threshold=2.0, use_cache="graph")
    assert not torch.equal(other[0], mel)  # (another seed: other prenet masks)
    eager = tts.generate_speech(src_tokens=tok, spkembs=spk, threshold=2.0, use_cache=True)
    assert eager[0].shape == mel.shape
    RT.dtype = torch.bfloat16


@pytest.mark.parametrize("dtype,tol", [(torch.float32, 2e-3), (torch.bfloat16, 6e-2)])
def test_speech_pretraining_branch_of_forward(cuda, dtype, tol):
    """models/speecht5.py:813-961 with target_list on the device: prenet with label alignment + feature penalty ->
    encoder -> masked-prediction head (speech_encoder_postnet.py:76-124), Gumbel quantizer + code mixing (:858-882),
    speech decoder on the mixed states; against the same composition of the CPU oracles with the same Gumbel noise and
    time permutation (SURVEY 8a row 22)."""
    from oracle import pretrain_oracle as P
    from oracle import speecht5_oracle as OT
    from oracle import speecht5_oracle_asr as O
    from speecht5_b200.models import T5TransformerModel, make_args
    from speecht5_b200.ops import RT
    RT.dtype = dtype
    RT.manual_seed(1)
    RT.disable_device_seed()
    RT.clear_static()
    RT.invalidate_shadows()
    torch.manual_seed(11)
    over = dict(encoder_layers=2, decoder_layers=2, bert_init=True, mask_prob=0.0, mask_channel_prob=0.0, dropout=0.0,
                attention_dropout=0.0, activation_dropout=0.0, dprenet_dropout_rate=0.0, postnet_dropout_rate=0.0,
                transformer_enc_positional_dropout_rate=0.0, transformer_dec_positional_dropout_rate=0.0,
                encoder_layerdrop=0.0, decoder_layerdrop=0.0, feature_grad_mult=1.0)
    oargs = O.base_asr_args(**over)
    tts = OT.T5TransformerModelOracle(oargs).train()
    prenet = O.SpeechEncoderPrenet(oargs).train()
    d = oargs.encoder_embed_dim
    head = P.SpeechEncoderPostnet([23], encoder_embed_dim=d, final_dim=32).train()
    quant = P.GumbelVectorQuantizer(dim=d, num_vars=10, groups=2, vq_dim=d).train()
    args = make_args("t5_transformer_base_asr", build_speech_encoder=True, use_conv_pos=True, use_sinc_pos=True,
                     use_codebook=True, latent_vars=10, latent_groups=2, codebook_prob=0.5, hubert_num_classes=[23],
                     final_dim=32, **over)
    model = T5TransformerModel.build_model(args).to(cuda).train()
    sd = {k: v for k, v in tts.state_dict().items() if not k.startswith("text_encoder_prenet.")}
    for k, v in prenet.state_dict().items():
        k = {"pos_conv_g": "pos_conv.0.weight_g", "pos_conv_v": "pos_conv.0.weight_v", "pos_conv_bias": "pos_conv.0.bias"}.get(k, k)
        sd["speech_encoder_prenet." + k] = v
    sd.update({"hubert_layer." + k: v for k, v in head.state_dict().items()})
    sd.update({"quantizer." + k: v for k, v in quant.state_dict().items()})
    model.load_state_dict(sd)
    B, n = 2, 8000
    wave = torch.randn(B, n) * 0.3
    pad = torch.zeros(B, n, dtype=torch.bool)
    pad[1, 7000:] = True
    with torch.no_grad():
        T = prenet(wave, pad, None, None)[0].shape[1]
    labels = [torch.randint(0, 23, (B, T + 3))]
    mask_idx = torch.zeros(B, T, dtype=torch.bool)
    mask_idx[0, 2:9] = True
    mask_idx[1, 4:11] = True
    prev, tgt_lengths, spk = torch.randn(B, 9, 80), torch.tensor([9, 7]), torch.randn(B, 512)
    noise = -torch.empty(B * T * 2, 10).exponential_().log()
    perm = torch.randperm(T)
    with torch.no_grad():
        x_ref, enc_pad, fpen_ref = prenet(wave, pad, mask_idx, None)
        enc = tts.encoder(x_ref, enc_pad)
        enc_btc = enc["encoder_out"][0].transpose(0, 1)
        hub_ref = head(enc_btc, enc_pad, mask_idx, [labels[0][:, :T]])
        q = quant(enc_btc, noise)
        enc["encoder_out"] = [P.mix_codes(enc_btc, q["x"], 0.5, perm).transpose(0, 1)]
        dec_in, tgt_mask = tts.speech_decoder_prenet(prev, tgt_lengths, spk)
        dec_out, _ = tts.decoder(dec_in, tgt_mask, enc, alignment_layer=None)
        before_ref, after_ref, logits_ref = tts.speech_decoder_postnet(dec_out)
    model._gumbel_noise, model._codebook_perm = noise.to(cuda), perm.to(cuda)
    hub, (before, after, logits, attn) = model(
        source=wave.to(cuda), padding_mask=pad.to(cuda), prev_output_tokens=prev.to(cuda),
        tgt_lengths=tgt_lengths.to(cuda), spkembs=spk.to(cuda), target_list=[labels[0].to(cuda)],
        task_name="speech_pretrain", mask_indices=mask_idx.to(cuda))

    def close(a, b, t):
        a, b = torch.as_tensor(a).detach().cpu().double(), torch.as_tensor(b).double()
        fin = torch.isfinite(b)
        return torch.equal(torch.isfinite(a), fin) and ((a[fin] - b[fin]).norm() / b[fin].norm().clamp_min(1e-12)).item() < t
    assert close(hub["features_pen"], fpen_ref, tol)
    assert close(hub["logit_m_list"][0], hub_ref["logit_m_list"][0], 4 * tol)
    assert close(hub["logit_u_list"][0], hub_ref["logit_u_list"][0], 4 * tol)
    assert close(hub["prob_perplexity"], q["prob_perplexity"], tol) and hub["num_vars"] == q["num_vars"]
    if dtype == torch.float32:  # bf16: a flipped arg-max of the Gumbel draw swaps a whole code vector; fp32 only
        assert close(after, after_ref, tol) and close(before, before_ref, tol) and close(logits, logits_ref, 3 * tol)
    # the whole branch is differentiable end to end: reconstruction + head losses reach the waveform filters
    loss = after.float().square().mean() + sum(x.float().logsumexp(-1).mean() for x in hub["logit_m_list"]) + hub["features_pen"]
    loss.backward()
    g = model.speech_encoder_prenet.feature_extractor.conv_layers[0][0].weight.grad
    assert g is not None and torch.isfinite(g).all() and g.abs().sum() > 0
    assert torch.isfinite(model.quantizer.vars.grad).all() and torch.isfinite(model.hubert_layer.label_embs_concat.grad).all()
    if dtype == torch.float32:
        # the speech pre-training CRITERION (pinned to the reference's own in tests/test_ref_pin_cpu.py) through the
        # dispatcher on the device model, against the same criterion fed with the oracle composition's outputs
        from speecht5_b200.criterions import SpeechPretrainCriterion, SpeechT5Criterion
        L = 2 * prev.shape[1]
        olens = 2 * tgt_lengths
        stop = torch.zeros(B, L)
        for b_ in range(B):
            stop[b_, int(olens[b_]) - 1:] = 1.0
        sample = {"id": torch.arange(B), "task_name": "speech_pretrain", "target_list": [labels[0]],
                  "labels": stop, "dec_target": torch.randn(B, L, 80), "dec_target_lengths": olens,
                  "src_lengths": torch.tensor([T, T]),
                  "net_input": dict(source=wave, padding_mask=pad, prev_output_tokens=prev, tgt_lengths=tgt_lengths,
                                    spkembs=spk, task_name="speech_pretrain", mask_indices=mask_idx)}

        class OracleOutputs(torch.nn.Module):
            reduction_factor = 2
            get_logits, get_targets, get_extra_losses = (T5TransformerModel.get_logits, T5TransformerModel.get_targets,
                                                         T5TransformerModel.get_extra_losses)

            def forward(self, target_list=None, **ni):
                out = dict(hub_ref, features_pen=fpen_ref, **{k: q[k] for k in ("prob_perplexity", "code_perplexity", "num_vars")})
                return out, (before_ref, after_ref, logits_ref, None)

        kw = dict(pred_masked_weight=1.0, pred_nomask_weight=0.5, loss_weights=[10.0, 0.1], hubert_weight=1.0, dec_weight=0.5)
        want, n_want, log_want = SpeechPretrainCriterion(None, True, **kw)(OracleOutputs(), sample)
        dev_sample = {k: (v.to(cuda) if torch.is_tensor(v) else v) for k, v in sample.items()}
        dev_sample["target_list"] = [labels[0].to(cuda)]
        dev_sample["net_input"] = {k: (v.to(cuda) if torch.is_tensor(v) else v) for k, v in sample["net_input"].items()}
        model.zero_grad()
        got, n_got, log_got = SpeechT5Criterion(None, **kw)(model, dev_sample)
        assert n_got == n_want and set(log_got) == set(log_want)
        assert abs(got.item() - want.item()) < 5e-3 * abs(want.item()), (got.item(), want.item())
        for k in ("loss_m_0", "loss_u_0", "dec_loss", "l1_loss", "bce_loss", "loss_features_pen", "loss_prob_perplexity"):
            assert abs(log_got[k] - log_want[k]) < 1e-2 * max(1.0, abs(log_want[k])), (k, log_got[k], log_want[k])
        (got / n_got).backward()
        assert torch.isfinite(model.speech_encoder_prenet.feature_extractor.conv_layers[0][0].weight.grad).all()
    RT.dtype = torch.bfloat16


@pytest.mark.parametrize("C,k,s,n,dtype", [(512, 10, 5, 4000, torch.float32), (512, 10, 5, 16000, torch.bfloat16),
                                           (32, 10, 5, 1203, torch.float32), (96, 16, 4, 999, torch.float32),
                                           (258, 7, 3, 2000, torch.bfloat16)])
def test_layer0_layer_norm_kernels_against_torch(cuda, C, k, s, n, dtype):
    """st5_conv0_ln_gelu_fwd / _bwd (layer 0 of the "layer_norm" extractor: conv + per-frame LayerNorm + GELU in one
    pass; speech_encoder_prenet.py:308-318) against the same statement in torch fp64 autograd: output, saved
    statistics, and the accumulated dw / dgamma / dbeta. Widths: the real 512, the tiny fixtures' 32, a channel count
    that is not a multiple of 64, more than 10 taps (the 8-taps-per-warp instantiation)."""
    from speecht5_b200 import kernels as K
    from speecht5_b200.ops import _resolve_act
    g = torch.Generator().manual_seed(C + n)
    B = 3
    wave = (torch.randn(B, n, generator=g) * 0.2).to(cuda)
    w = (torch.randn(C, k, generator=g) * (2.0 / k) ** 0.5).to(cuda)
    gamma = (1 + 0.2 * torch.randn(C, generator=g)).to(cuda)
    beta = (0.2 * torch.randn(C, generator=g)).to(cuda)
    T0 = (n - k) // s + 1
    act = _resolve_act("gelu", dtype)
    y = torch.empty(B, T0, C, dtype=dtype, device=cuda)
    mean = torch.empty(B * T0, device=cuda)
    rstd = torch.empty_like(mean)
    K.conv0_ln_gelu_fwd(wave, w, gamma, beta, y, mean, rstd, s, 1e-5, act)
    w64, g64, b64 = (t.double().clone().requires_grad_() for t in (w, gamma, beta))
    v = torch.nn.functional.conv1d(wave.double()[:, None], w64[:, None], stride=s).transpose(1, 2)
    want = torch.nn.functional.gelu(torch.nn.functional.layer_norm(v, (C,), g64, b64, 1e-5))
    tol = 2e-5 if dtype == torch.float32 else 6e-3
    assert rel(y, want.detach()) < tol
    assert rel(mean, v.detach().mean(-1).reshape(-1)) < 1e-5
    assert rel(rstd, (v.detach().var(-1, unbiased=False) + 1e-5).rsqrt().reshape(-1)) < 1e-5
    dy = torch.randn(B, T0, C, generator=g).to(cuda).to(dtype)
    gw, gg, gb = torch.autograd.grad(want, (w64, g64, b64), dy.double())
    dw = torch.full_like(w, 0.5)  # (accumulated into what is there)
    dg, db = torch.zeros(C, device=cuda), torch.zeros(C, device=cuda)
    K.conv0_ln_gelu_bwd(dy, wave, w, gamma, beta, mean, rstd, dw, dg, db, s, act)
    gtol = 1e-4 if dtype == torch.float32 else 2e-2  # (bf16 mode differentiates the tanh form of GELU)
    assert rel(dw - 0.5, gw) < gtol and rel(dg, gg) < gtol and rel(db, gb) < gtol
    # stand-alone GELU of the later layers (odd element count: vector body + scalar tail)
    z = torch.randn(7, 331, generator=g).to(cuda).to(dtype)
    out = torch.empty_like(z)
    K.act_fwd(z, out, act)
    assert rel(out, torch.nn.functional.gelu(z.double())) < (1e-6 if dtype == torch.float32 else 6e-3)


@pytest.mark.parametrize("dtype,tol,gtol", [(torch.float32, 1e-4, 2e-3), (torch.bfloat16, 3e-2, 0.2)])
def test_layer_norm_extractor_real_width_against_oracle(cuda, dtype, tol, gtol):
    """ConvFeatureExtractor(mode="layer_norm") at the real seven layers x 512 channels on 0.5 s of audio: output and
    every parameter gradient against the oracle's ConvFeatureExtractionModel (pinned to the reference's in this mode)."""
    import re
    from oracle.speecht5_oracle_asr import CONV_FEATURE_LAYERS, ConvFeatureExtractionModel
    from speecht5_b200 import frontend
    from speecht5_b200.ops import RT
    RT.dtype = dtype
    RT.clear_static()
    RT.invalidate_shadows()
    torch.manual_seed(21)
    ref = ConvFeatureExtractionModel(CONV_FEATURE_LAYERS, "layer_norm", False).double()
    for blk in ref.conv_layers:
        torch.nn.init.normal_(blk[2].weight, 1.0, 0.2), torch.nn.init.normal_(blk[2].bias, 0.0, 0.2)
    mine = frontend.ConvFeatureExtractor(CONV_FEATURE_LAYERS, "layer_norm", False)
    to_ref = lambda k: re.sub(r"^(conv_layers\.\d+\.2)\.", r"\1.1.", k)  # noqa: E731
    mine.load_state_dict({to_ref(k): v.float() for k, v in ref.state_dict().items()})
    mine = mine.to(cuda)
    wave = torch.randn(2, 8000, dtype=torch.float64) * 0.3
    want = ref(wave).transpose(1, 2)
    got = mine(wave.float().to(cuda))
    assert got.shape == want.shape and got.dtype == dtype and rel(got.cpu(), want.detach()) < tol
    probe = torch.randn_like(want)
    (want * probe).sum().backward()
    (got.float() * probe.float().to(cuda)).sum().backward()
    named = dict(mine.named_parameters())
    for k, p in ref.named_parameters():
        g = named[to_ref(k)].grad
        assert g is not None and rel(g.cpu(), p.grad) < gtol, (k, rel(g.cpu(), p.grad))
    RT.dtype = torch.bfloat16


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_joint_pretraining_update_through_the_trainer(cuda, dtype):
    """BASELINE config 4 in miniature on the device: t5_transformer_large's structure (layer_norm extractor, pre-LN, tied
    embeddings, masked-prediction head, shared quantizer) at tiny widths; a speech_pretrain + a text_pretrain micro-batch
    per update through B200Trainer (these updates run eagerly, graphs on or off). Loss falls, parameters move, no
    graph is captured. (tests/test_frontend_cpu.py runs the same on emulated kernels.)"""
    import numpy as np
    from helpers import NO_DROPOUT, TINY
    from speecht5_b200.criterions import SpeechT5Criterion
    from speecht5_b200.data import synthetic_speech_pretrain_batch, synthetic_text_pretrain_batch
    from speecht5_b200.models import make_args
    from speecht5_b200.ops import RT
    from speecht5_b200.tasks import SpeechT5Task
    from speecht5_b200.trainer import B200Trainer
    RT.dtype = dtype
    RT.manual_seed(3)
    RT.clear_static()
    RT.invalidate_shadows()
    torch.manual_seed(5)
    np.random.seed(5)
    V = 40
    args = make_args("t5_transformer_large", **dict(TINY, **NO_DROPOUT), bert_init=True, build_speech_encoder=True,
                     build_text_decoder=True, share_input_output_embed=True, use_codebook=True, latent_vars=10,
                     latent_groups=2, codebook_prob=0.5, hubert_num_classes=[23], final_dim=16, vocab_size=V,
                     conv_feature_layers="[(32, 10, 5)] + [(32, 3, 2)] * 4 + [(32, 2, 2)] * 2", conv_pos=16,
                     conv_pos_groups=4, mask_prob=0.5, hubert_mask_length=3, max_text_positions=600)
    task = SpeechT5Task(args)
    model = task.build_model(args).to(cuda).train()
    crit = SpeechT5Criterion(task, loss_weights=[10.0], dec_weight=0.5, bart_weight=1.0, hubert_weight=1.0)
    tr = B200Trainer(model, crit, task, lr=2e-3, clip_norm=10.0, use_cuda_graph=True)
    speech = synthetic_speech_pretrain_batch(2, 6400, n_classes=23, seed=1, pin=True)
    text = synthetic_text_pretrain_batch(3, 12, V, mask_idx=V - 2, seed=2, pin=True)
    before = {n: p.detach().clone() for n, p in model.named_parameters()}
    losses = []
    for _ in range(8):
        out, stats = tr.train_step([speech, text])
        assert stats is None and out.shape == (2,) and bool(torch.isfinite(out).all())
        losses.append(out.tolist())
    tr.check_overflow()  # (raises if an update was skipped for a non-finite gradient norm)
    assert tr.graph_misses == 0 and tr.num_updates == 8
    assert losses[-1][0] < losses[0][0] and losses[-1][1] < losses[0][1], losses
    moved = {n for n, p in model.named_parameters() if not torch.equal(p.detach(), before[n])}
    for key in ("speech_encoder_prenet.feature_extractor.conv_layers.0.0.weight",
                "speech_encoder_prenet.feature_extractor.conv_layers.3.2.1.weight", "hubert_layer.label_embs_concat",
                "quantizer.vars", "encoder.layers.0.fc1.weight", "decoder.layers.0.encoder_attn.k_proj.weight"):
        assert key in moved, key
    RT.dtype = torch.bfloat16
    RT.clear_static()
    RT.invalidate_shadows()
