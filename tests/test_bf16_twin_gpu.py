"""-m gpu: throughput mode (RT.dtype = bf16) against the reference model's own bf16 run, at Base widths.

Every output, loss term and parameter gradient of the product model P must be no further from an fp64 run R of the
oracle than C = 2 times the distance of the oracle's bf16 twin T, plus a relative floor F = 2^-12 (tests/bf16_twin.py).
The model-level bounds elsewhere (6e-2 on outputs, 0.25 on gradients) pin the reference's fixtures; they cannot see a
gradient 6 % off for one parameter or one utterance's key mask off by one. This module can, and its sensitivity test
shows it: each injected composition fault above the twin's own noise fails the check.

Base widths (d = 768, 12 heads, FFN 3072, relative positions +-160), 2 + 2 layers, attention sharpened (q, k and the
relative-position table x6) as in test_model_gpu.test_base_dims_against_oracle, dropout off. Ragged batches; the TTS and
text cases have an utterance of one token. Run with -s for the worst ratio per check."""
import time

import pytest
import torch

import bf16_twin as TW
from helpers import NO_DROPOUT, rel, to_device

pytestmark = pytest.mark.gpu
PAD = 1


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    t0 = time.time()
    yield
    _CACHE.clear()  # (T / R outputs and fp64 gradients of the t2s cases, kept on the device across this module's tests)
    TW.print_report()
    print(f"bf16 twin module: {time.time() - t0:.1f} s")


@pytest.fixture(autouse=True)
def _switches():
    from speecht5_b200.ops import RT
    keep = (RT.dtype, RT.attn_fused, RT.probs_grad_heads)
    yield
    RT.dtype, RT.attn_fused, RT.probs_grad_heads = keep
    RT.clear_static()
    RT.invalidate_shadows()
    torch.cuda.synchronize()


def _build(dev, **over):
    from speecht5_b200.models import T5TransformerModel, make_args
    from speecht5_b200.ops import RT
    RT.dtype = torch.bfloat16
    RT.manual_seed(1)
    RT.disable_device_seed()
    RT.clear_static()
    RT.invalidate_shadows()
    return T5TransformerModel.build_model(make_args("t5_transformer_base_asr", **over)).to(dev).train()


def _sharpen(oracle, seed_ln=False, cross=6.0):
    """Peaky attention as in test_base_dims_against_oracle: q / k projections and the relative-position table x6; the
    cross-attention's q / k projections x `cross`."""
    with torch.no_grad():
        for n, p in oracle.named_parameters():
            if n.endswith("alpha"):
                p.fill_(0.9)
            elif "q_proj.weight" in n or "k_proj.weight" in n or "pe_k" in n:
                p.mul_(cross if "encoder_attn" in n else 6.0)
            elif seed_ln and ("norm_k" in n or "layer_norm" in n):
                p.add_(torch.randn_like(p) * 0.1)


def _oracle_run(m, dev, fn):
    """Run `fn(m)` with factory functions on `dev` (the oracle builds masks, positions and tables without a device)."""
    with torch.device(dev):
        return fn(m)


def _grads(model, rename=None):
    return TW.param_grads(model, rename)


# ------------------------------------------------------------------------------------------------------ t2s
T2S = dict(encoder_layers=2, decoder_layers=2, bert_init=True, **NO_DROPOUT)
T2S_PRELN = dict(T2S, layer_norm_first=True, decoder_normalize_before=True)
_CACHE = {}


def _t2s_batch(B, T_txt, T_mel, seed):
    """oracle.synthetic_tts_batch with the last utterance cut to one text token and 4 mel frames (2 decoder steps)."""
    from oracle.speecht5_oracle import synthetic_tts_batch
    s = synthetic_tts_batch(B, T_txt, T_mel, seed=seed)
    ni = s["net_input"]
    b = B - 1
    ni["src_tokens"][b, 1:] = PAD
    ni["src_lengths"][b] = 1
    fb = s["dec_target"]
    fb[b, 4:] = 0.0
    s["dec_target_lengths"][b] = 4
    s["labels"][b] = (torch.arange(T_mel) >= 3).float()
    fb_in = fb[:, 1::2]
    ni["prev_output_tokens"] = torch.cat([fb_in.new_zeros((B, 1, fb.shape[2])), fb_in[:, :-1]], dim=1).contiguous()
    ni["tgt_lengths"] = torch.div(s["dec_target_lengths"], 2, rounding_mode="floor")
    s["src_lengths"] = ni["src_lengths"]
    s["target"] = fb
    s["ntokens"] = int(ni["src_lengths"].sum())
    return TW.round_tree(s)


def _t2s_inputs(over, B, T_txt, T_mel, seed, cross=6.0):
    from oracle.speecht5_oracle import T5TransformerModelOracle, base_args
    torch.manual_seed(seed)
    oracle = T5TransformerModelOracle(base_args(**over)).train()
    _sharpen(oracle, seed_ln=over.get("layer_norm_first", False), cross=cross)
    state = TW.round_tree({k: v.clone() for k, v in oracle.state_dict().items()})
    return state, _t2s_batch(B, T_txt, T_mel, seed)


def _t2s_oracle_arms(dev, over, state, sample):
    """T and R: outputs (dict), loss terms (list) and parameter gradients of one update."""
    from oracle.speecht5_oracle import T5TransformerModelOracle, base_args, tts_loss
    arms = []
    for m in TW.twin_and_reference(lambda: T5TransformerModelOracle(base_args(**over)).train(), state, dev):
        dt = next(m.parameters()).dtype
        loss_dt = torch.float32 if dt == torch.bfloat16 else torch.float64
        ni = TW.cast_tree(sample["net_input"], dt, dev)
        s = TW.cast_tree(sample, loss_dt, dev)
        scales = TW.alpha_scales(m)

        def run(mm):
            before, after, logits, attn = mm(**ni)
            out = [before.to(loss_dt), after.to(loss_dt), logits.to(loss_dt), [a.to(loss_dt) for a in attn]]
            terms = tts_loss(out, s)
            terms[0].backward()
            return out, terms
        out, terms = _oracle_run(m, dev, run)
        outs = dict(before=out[0], after=out[1], logits=out[2])
        outs.update({f"cross-attn layer {i}": a.transpose(1, 2) for i, a in enumerate(out[3])})  # [B, Tq, H, Tk]
        arms.append(({k: v.detach() for k, v in outs.items()}, [t.detach() for t in terms], _grads(m), scales))
        del m
    return arms


def _t2s_product(dev, over, state, sample, heads=2, fault=None):
    """P: the plain product model (no trainer) in throughput mode; guided attention differentiates the first `heads`
    heads of the returned maps (RT.probs_grad_heads, the hint the trainer gives the attention backward)."""
    from speecht5_b200.criterions import TexttoSpeechLoss
    from speecht5_b200.ops import RT
    model = _build(dev, **over)
    model.load_state_dict(state)
    if fault is not None:
        fault(model)
    RT.probs_grad_heads = heads
    s = to_device(sample, dev)
    before, after, logits, attn = model(**s["net_input"])
    terms = TexttoSpeechLoss(None, use_guided_attn_loss=True).compute_loss(model, (before, after, logits, attn), s)
    terms[0].backward()
    RT.probs_grad_heads = 0
    outs = dict(before=before, after=after, logits=logits)
    outs.update({f"cross-attn layer {i}": a.transpose(1, 2) for i, a in enumerate(attn)})
    out = ({k: v.detach().float() for k, v in outs.items()}, [t.detach().float() for t in terms], _grads(model))
    del model
    return out


def _t2s_compare(tw, P, T, R, sample):
    (op, lp, gp), (ot, lt, gt, _), (orr, lr, gr, scales) = P, T, R
    mel = sample["dec_target_lengths"]
    steps = sample["net_input"]["tgt_lengths"]
    for k in orr:
        rows = mel if k in ("before", "after", "logits") else steps
        tw.tensor(k, op[k], ot[k], orr[k], rows=rows)
    for name, a, b, c in zip(("loss", "l1", "l2", "bce", "guided attn"), lp, lt, lr):
        tw.scalar(f"loss {name}", a, b, c)
    n = tw.grads(gp, gt, gr, scalar_abs=scales)
    assert n > 40, n


def _t2s_reference(dev, case):
    """(over, state, sample, (T, R)) of one entry of T2S_CASES, computed once per module."""
    if case not in _CACHE:
        over, B, T_txt, T_mel, seed, cross = T2S_CASES[case]
        state, sample = _t2s_inputs(over, B, T_txt, T_mel, seed, cross)
        _CACHE[case] = (over, state, sample, _t2s_oracle_arms(dev, over, state, sample))
    return _CACHE[case]


T2S_CASES = {
    # encoder T = 45: the relative-position resident kernel (forward + fused backward with the head-major dQP scatter)
    "t2s post-LN T=45": (T2S, 3, 45, 64, 3, 6.0),
    # encoder T = 200 > 160: the streaming kernel with clipped relative positions; cross-attention over 200 keys
    "t2s post-LN T=200": (T2S, 3, 200, 96, 5, 6.0),
    "t2s pre-LN T=45": (T2S_PRELN, 3, 45, 64, 7, 6.0),
}
# the T = 45 case with the cross-attention q / k projections x2 instead of x6: a softmax far from saturation, where a
# scale error moves the maps (at x6 the maps are nearly one-hot and a 6 % scale error moves them by 0.8 of T's error)
SENSITIVITY_CASES = {"t2s post-LN T=45 cross x2": (T2S, 3, 45, 64, 3, 2.0)}
T2S_CASES.update(SENSITIVITY_CASES)


@pytest.mark.parametrize("case", [c for c in T2S_CASES if c not in SENSITIVITY_CASES])
def test_t2s_update_against_the_bf16_twin(cuda, case):
    over, state, sample, (T, R) = _t2s_reference(cuda, case)
    P = _t2s_product(cuda, over, state, sample)
    tw = TW.Twin(case)
    _t2s_compare(tw, P, T, R, sample)
    print("\n" + tw.verdict())
    tw.assert_ok()


def test_t2s_unfused_tensor_core_route_against_the_bf16_twin(cuda):
    """RT.attn_fused = False: QK^T / Q.PE^T / PV on the GEMM with the softmax row kernel, and the unfused backward with
    the relative-position table gradient summed over (utterance, head) parts."""
    from speecht5_b200.ops import RT
    case = "t2s post-LN T=45"
    over, state, sample, (T, R) = _t2s_reference(cuda, case)
    RT.attn_fused = False
    P = _t2s_product(cuda, over, state, sample)
    tw = TW.Twin("t2s unfused route T=45")
    _t2s_compare(tw, P, T, R, sample)
    print("\n" + tw.verdict())
    tw.assert_ok()


def test_t2s_trainer_graph_replay_against_the_bf16_twin(cuda):
    """The T = 45 update through B200Trainer as a replayed CUDA graph: the flat-buffer gradients (fp.grads at
    fp.offsets) under the same per-parameter bound."""
    from speecht5_b200.criterions import SpeechT5Criterion
    from speecht5_b200.models import make_args
    from speecht5_b200.ops import RT
    from speecht5_b200.tasks import SpeechT5Task
    from speecht5_b200.trainer import B200Trainer
    case = "t2s post-LN T=45"
    over, state, sample, (T, R) = _t2s_reference(cuda, case)
    RT.dtype = torch.bfloat16
    RT.clear_static()
    RT.disable_device_seed()
    args = make_args("t5_transformer_base_asr", **over)
    task = SpeechT5Task(args)
    model = task.build_model(args).to(cuda).train()
    model.load_state_dict(state)
    RT.invalidate_shadows()
    tr = B200Trainer(model, SpeechT5Criterion(task, use_guided_attn_loss=True), task, lr=0.0, use_cuda_graph=True)
    losses = tr.train_step([to_device(sample, cuda)])[0]
    torch.cuda.synchronize()
    assert tr.graph_misses == 1
    fp = tr.fp
    names = {id(p): n for n, p in model.named_parameters()}
    gp = {names[id(p)]: fp.grads[fp.offsets[id(p)]:fp.offsets[id(p)] + p.numel()].view(p.shape).clone()
          for p in fp.params}
    tw = TW.Twin("t2s trainer graph T=45")
    tw.scalar("loss", float(torch.as_tensor(losses).reshape(-1)[0]), T[1][0], R[1][0])
    assert tw.grads(gp, T[2], R[2], scalar_abs=R[3]) > 40
    del tr, model
    print("\n" + tw.verdict())
    tw.assert_ok()


# ------------------------------------------------------------------------------------------------------ sensitivity
def _fault_key_mask(model, monkeypatch):
    """The encoder self-attention masks the last valid key of utterance 0 (a key mask lost to an off-by-one)."""
    from speecht5_b200 import ops
    inner = ops.attention

    def attention(q_buf, kv_buf, **kw):
        if kw.get("pe_k") is not None and kw.get("key_pad") is not None:
            kp = kw["key_pad"].clone()
            n = int((~kp[0]).sum())
            kp[0, n - 1] = True
            kw["key_pad"] = kp
        return inner(q_buf, kv_buf, **kw)
    monkeypatch.setattr(ops, "attention", attention)


def _fault_bias_grad(model, monkeypatch):
    """One layer's out_proj bias gradient scaled by 1 - 2^-4."""
    b = model.decoder.layers[1].self_attn.out_proj.bias
    b.register_hook(lambda g: g * (1.0 - 2.0 ** -4))


def _fault_table_share(model, monkeypatch):
    """The shared relative-position table loses encoder layer 0's contribution to its gradient."""
    from speecht5_b200 import ops
    inner = ops.attention
    seen = []

    def attention(q_buf, kv_buf, **kw):
        if kw.get("pe_k") is not None and not seen:
            seen.append(1)
            kw["pe_k"] = kw["pe_k"].detach()
        return inner(q_buf, kv_buf, **kw)
    monkeypatch.setattr(ops, "attention", attention)


def _cross_scale(k):
    """The cross-attention route runs with its softmax scale multiplied by 1 + 2^-k (both decoder layers)."""
    def fault(model, monkeypatch):
        from speecht5_b200 import ops
        inner = ops.attention

        def attention(q_buf, kv_buf, **kw):
            if kv_buf is not None:
                fault.hits += 1
                kw["scale"] = kw["scale"] * (1.0 + 2.0 ** -k)
            return inner(q_buf, kv_buf, **kw)
        monkeypatch.setattr(ops, "attention", attention)
    fault.hits = 0
    return fault


FAULTS = {"key mask of one utterance's last valid key": _fault_key_mask,
          "out_proj bias gradient x (1 - 2^-4)": _fault_bias_grad,
          "one layer's share of the relative-position table gradient dropped": _fault_table_share}
FAULTS.update({f"cross-attention scale x (1 + 2^-{k})": _cross_scale(k) for k in (5, 7)})
# (fault, case, detectable). A scale error of 2^-7 is NOT detectable by this standard, and the test shows why: it moves
# the cross-attention maps by less than the twin's own distance from fp64 (|P_fault - P| / |T - R| measured 0.22 at x6,
# 0.62 at x2 on an H100). With P's own error e0 ~ 0.5 e_T, failing (1) needs a shift f with e0^2 + f^2 > (C e_T)^2,
# f > 1.9 e_T; even C = 1 would need f > 0.87 e_T. Such a fault is smaller than what the reference's own bf16 run does
# to the same maps. The shift grows linearly with the error: 2^-5 moves them by 2.35 e_T and fails.
FAULT_CASES = [(f, "t2s post-LN T=45", True) for f in list(FAULTS)[:3]] + [
    ("cross-attention scale x (1 + 2^-5)", "t2s post-LN T=45 cross x2", True),
    ("cross-attention scale x (1 + 2^-7)", "t2s post-LN T=45", False),
    ("cross-attention scale x (1 + 2^-7)", "t2s post-LN T=45 cross x2", False)]


@pytest.mark.parametrize("fault,case,detectable", FAULT_CASES)
def test_twin_check_flags_small_composition_faults(cuda, monkeypatch, fault, case, detectable):
    """Each detectable fault, injected in Python on the plain model, fails the twin check. Printed: the worst e_P /
    bound, and whether the loose model-level bounds (outputs 6e-2, gradients 0.25 relative to fp64) would flag it. A
    scale fault must reach both cross-attention calls and move the maps; one below the twin's noise (see FAULT_CASES)
    must move them by less than T's own error."""
    over, state, sample, (T, R) = _t2s_reference(cuda, case)
    P = _t2s_product(cuda, over, state, sample, fault=lambda m: FAULTS[fault](m, monkeypatch))
    monkeypatch.undo()
    if hasattr(FAULTS[fault], "hits"):
        assert FAULTS[fault].hits == 2, FAULTS[fault].hits  # the route of both decoder layers took the fault
        FAULTS[fault].hits = 0
        clean = _t2s_product(cuda, over, state, sample)
        live = max(rel(P[0][k], clean[0][k]) / rel(T[0][k], R[0][k]) for k in P[0] if k.startswith("cross"))
        print(f"\n{fault} on {case}: largest map shift |P_fault - P| / |T - R| = {live:.3g}")
        assert live > 0.1, live  # the injection reached the route
        if not detectable:
            assert live < 1.0, f"{fault} moves the maps by {live:.3g} of the twin's error: it should be detectable"
            return
    tw = TW.Twin(f"fault: {fault}", report=False)
    _t2s_compare(tw, P, T, R, sample)
    out_rel = max(rel(P[0][k], R[0][k]) for k in ("before", "after"))
    gmax = max(float(g.norm()) for g in R[2].values() if g is not None)
    grad_rel = max(rel(P[2][n], g) for n, g in R[2].items() if g is not None and float(g.norm()) > 1e-4 * gmax)
    loose = out_rel >= 6e-2 or grad_rel >= 0.25
    print(f"\nfault '{fault}' on {case}: worst e_P / bound {tw.worst:.3g} ({tw.worst_what}); loose bounds: mel rel {out_rel:.3g}, "
          f"worst grad rel {grad_rel:.3g} -> {'flagged' if loose else 'not flagged'}; failed checks: "
          + ", ".join(f"{w} {q:.3g}" for w, q in sorted(tw.fails, key=lambda f: -f[1])[:8]))
    TW.REPORT[f"sensitivity: {fault}, {case} (must be > 1)"] = tw.worst
    assert tw.fails, f"the twin check missed the fault: {tw.verdict()}"


# ------------------------------------------------------------------------------------------------------ cached decoding
def _cached_steps(model, enc, dec_in, steps, need_attn):
    """Teacher-forced incremental.decoder_step in its device-step form (the form the captured synthesis graphs replay):
    row t of the key/value cache written by index_copy_, self-attention over a bucketed span of cache rows (16, 32,
    64, ...) with the rows past t masked, cross-attention with the encoder's key padding. dec_in [B, T, C] is the
    prenet output of the whole target, fed one position per step. Returns ([B, T, C] outputs, [B, T, H, S] maps)."""
    from speecht5_b200.incremental import DecoderCache, decoder_step
    B, dev = dec_in.shape[0], dec_in.device
    rows = 16
    while rows < steps:
        rows *= 2
    cache = DecoderCache(model.decoder, enc, rows)
    t_dev = torch.zeros(1, dtype=torch.int64, device=dev)
    pos = torch.arange(rows, device=dev)
    zs, maps = [], []
    for t in range(steps):
        span = 16
        while span < t + 1:
            span *= 2
        t_dev.fill_(t)
        self_pad = (pos[:span] > t_dev).to(torch.uint8)[None].expand(B, span).contiguous()
        z, la = decoder_step(model.decoder, dec_in[:, t:t + 1], cache, need_head_weights=need_attn, t_dev=t_dev,
                             span=span, self_pad=self_pad)
        zs.append(z)
        if need_attn:
            maps.append(torch.stack([a[:, :, 0, :] for a in la], 1))  # [B, layers, H, S]
    z = torch.cat(zs, 1)
    return z, (torch.stack(maps, 1) if need_attn else None)  # maps: [B, T, layers, H, S]


def test_teacher_forced_cached_speech_decoding_against_the_bf16_twin(cuda):
    """The speech decoder stepped through the key/value cache and the split-KV decode kernel over a fixed target (no
    feedback: the arms cannot diverge), each step against R's full-sequence decoder at that position. 40 steps cross
    the 16 / 32 / 64 span buckets; the encoder keys are padded for two of three utterances (one has one token)."""
    from oracle.speecht5_oracle import T5TransformerModelOracle, base_args
    over, B, T_txt, T_mel, seed = T2S, 3, 45, 80, 11
    state, sample = _t2s_inputs(over, B, T_txt, T_mel, seed)
    ni, steps = sample["net_input"], T_mel // 2
    arms = []
    for m in TW.twin_and_reference(lambda: T5TransformerModelOracle(base_args(**over)).eval(), state, cuda):
        x = TW.cast_tree(ni, next(m.parameters()).dtype, cuda)

        @torch.no_grad()
        def run(mm):
            enc = mm.encoder(*mm.text_encoder_prenet(x["src_tokens"]))
            dec_in, _ = mm.speech_decoder_prenet(x["prev_output_tokens"], None, x["spkembs"])
            z, extra = mm.decoder(dec_in, None, enc, alignment_layer=-1)
            before = mm.speech_decoder_postnet.feat_out(z)
            maps = torch.stack([a.transpose(1, 2) for a in extra["attn"][0]], 2)  # [B, T, layers, H, S]
            return z.double(), before.double(), maps.double()
        arms.append(_oracle_run(m, cuda, run))
        del m
    T, R = arms
    model = _build(cuda, **over).eval()
    model.load_state_dict(state)
    s = to_device(sample, cuda)["net_input"]
    with torch.no_grad():
        enc = model.forward_text_encoder(s["src_tokens"])
        dec_in, _ = model.speech_decoder_prenet(s["prev_output_tokens"], spkembs=s["spkembs"])
        z, maps = _cached_steps(model, enc, dec_in, steps, need_attn=True)
        before = torch.cat([model.speech_decoder_postnet.project(z[:, t:t + 1].contiguous())[0].reshape(B, 1, -1)
                            for t in range(steps)], 1)
    P = (z.double(), before.double(), maps.double())
    tw = TW.Twin("cached speech decoding")
    for what, i in (("decoder output", 0), ("feat_out", 1), ("cross-attn", 2)):
        tw.tensor(what, P[i], T[i], R[i])
        for t in range(steps):  # every step on its own: the whole batch at position t
            tw._record(f"{what} step {t}", TW.ratio(P[i][:, t], T[i][:, t], R[i][:, t]), f"{what} per step")
    print("\n" + tw.verdict())
    tw.assert_ok()


def test_teacher_forced_cached_text_decoding_against_the_bf16_twin(cuda):
    """The text decoder stepped through the key/value cache over fixed target tokens, each step's logits against R's
    full-sequence logits at that position; ragged sources (one of one token), one target padded after 10 tokens."""
    from oracle.speecht5_oracle_asr import T5TransformerModelT2TOracle, base_asr_args
    over = dict(encoder_layers=2, decoder_layers=2, share_input_output_embed=True, bert_init=True, **NO_DROPOUT)
    torch.manual_seed(23)
    oracle = T5TransformerModelT2TOracle(base_asr_args(**over))
    _sharpen(oracle)
    state = TW.round_tree({k: v.clone() for k, v in oracle.state_dict().items()})
    g = torch.Generator().manual_seed(6)
    B, Ts, Tt, V = 3, 37, 40, 81
    src = torch.randint(4, V, (B, Ts), generator=g)
    src[1, 29:] = PAD
    src[2, 1:] = PAD
    prev = torch.randint(4, V, (B, Tt), generator=g)
    prev[:, 0] = 2
    prev[2, 10:] = PAD
    rows = prev.ne(PAD).sum(1)
    src, prev = src.to(cuda), prev.to(cuda)
    arms = []
    for m in TW.twin_and_reference(lambda: T5TransformerModelT2TOracle(base_asr_args(**over)).eval(), state, cuda):
        @torch.no_grad()
        def run(mm):
            enc = mm.encoder(*mm.text_encoder_prenet(src))
            dec_in, mask = mm.text_decoder_prenet(prev)
            z, _ = mm.decoder(dec_in, mask, enc, alignment_layer=None)
            return z.double(), mm.text_decoder_postnet(z).double()
        arms.append(_oracle_run(m, cuda, run))
        del m
    T, R = arms
    model = _build(cuda, build_text_decoder=True, **over).eval()
    model.load_state_dict(state)
    with torch.no_grad():
        enc = model.forward_text_encoder(src)
        dec_in = model.text_decoder_prenet(prev)[0]
        z, _ = _cached_steps(model, enc, dec_in, Tt, need_attn=False)
        logits = model.text_decoder_postnet(z)
    P = (z.double(), logits.double())
    tw = TW.Twin("cached text decoding")
    for what, i in (("decoder output", 0), ("text logits", 1)):
        tw.tensor(what, P[i], T[i], R[i], rows=rows)
        for t in range(Tt):
            b = rows > t  # utterances whose target is still running at position t
            tw._record(f"{what} step {t}", TW.ratio(P[i][b, t], T[i][b, t], R[i][b, t]), f"{what} per step")
    print("\n" + tw.verdict())
    tw.assert_ok()


# ------------------------------------------------------------------------------------------------------ t2t
def test_t2t_update_against_the_bf16_twin(cuda):
    """Text encoder -> text decoder (causal self-attention), tied embedding, label-smoothed CE on fp32 logits."""
    import torch.nn.functional as F
    from oracle.speecht5_oracle_asr import T5TransformerModelT2TOracle, base_asr_args, label_smoothed_nll_loss
    over = dict(encoder_layers=2, decoder_layers=2, share_input_output_embed=True, bert_init=True, **NO_DROPOUT)
    torch.manual_seed(21)
    oracle = T5TransformerModelT2TOracle(base_asr_args(**over)).train()
    _sharpen(oracle)
    state = TW.round_tree({k: v.clone() for k, v in oracle.state_dict().items()})
    g = torch.Generator().manual_seed(5)
    B, Ts, Tt, V, eos = 3, 37, 30, 81, 2
    src = torch.randint(4, V, (B, Ts), generator=g)
    src[1, 29:] = PAD
    src[2, 1:] = PAD
    tgt = torch.randint(4, V, (B, Tt), generator=g)
    tgt[:, -1] = eos
    tgt[2, 9] = eos
    tgt[2, 10:] = PAD
    prev = torch.full_like(tgt, PAD)
    prev[:, 0] = eos
    prev[:, 1:] = tgt[:, :-1]
    prev[2, 10:] = PAD
    rows = tgt.ne(PAD).sum(1)

    def run(m, dt):
        (logits, _), _, _ = m(src_tokens=src.to(cuda), prev_output_tokens=prev.to(cuda))
        lp = F.log_softmax(logits.to(dt), dim=-1)
        loss = label_smoothed_nll_loss(lp.view(-1, V), tgt.to(cuda).view(-1), 0.1, PAD)[0]
        loss.backward()
        return logits.detach().to(dt), loss.detach()

    arms = []
    for m in TW.twin_and_reference(lambda: T5TransformerModelT2TOracle(base_asr_args(**over)).train(), state, cuda):
        dt = torch.float32 if next(m.parameters()).dtype == torch.bfloat16 else torch.float64
        scales = TW.alpha_scales(m)
        arms.append(_oracle_run(m, cuda, lambda mm: run(mm, dt)) + (_grads(m), scales))
    model = _build(cuda, build_text_decoder=True, **over)
    model.load_state_dict(state)
    P = run(model, torch.float32) + (_grads(model),)
    (T, R) = arms
    tw = TW.Twin("t2t")
    tw.tensor("text logits", P[0], T[0], R[0], rows=rows)
    tw.scalar("loss", P[1], T[1], R[1])
    assert tw.grads(P[2], T[2], R[2], scalar_abs=R[3]) > 40
    print("\n" + tw.verdict())
    tw.assert_ok()


# ------------------------------------------------------------------------------------------------------ s2t
def _to_oracle_names(grads):
    """The product keeps the reference's checkpoint names (weight-normed pos_conv.0.*, the layer_norm extractor's
    conv_layers.{i}.2.1.*); the oracle's differ."""
    from oracle.speecht5_oracle_asr import reference_to_oracle_keys
    return reference_to_oracle_keys(grads)


def _to_reference_names(state, extractor):
    import re
    out = {}
    for k, v in state.items():
        k = k.replace("pos_conv_g", "pos_conv.0.weight_g").replace("pos_conv_v", "pos_conv.0.weight_v")
        k = k.replace("pos_conv_bias", "pos_conv.0.bias")
        if extractor == "layer_norm":
            k = re.sub(r"(feature_extractor\.conv_layers\.\d+\.2)\.", r"\1.1.", k)
        out[k] = v
    return out


@pytest.mark.parametrize("extractor", ["default", "layer_norm"])
def test_s2t_update_against_the_bf16_twin(cuda, extractor):
    """A 10 s waveform (~499 encoder frames: self- and cross-attention take the streaming kernels), CE + CTC, gradients
    down to conv layer 0; GroupNorm ("default") and per-conv LayerNorm ("layer_norm") front ends."""
    from oracle import speecht5_oracle_asr as O
    from speecht5_b200.criterions import SpeechT5Criterion
    over = dict(encoder_layers=2, decoder_layers=2, bert_init=True, mask_prob=0.0, mask_channel_prob=0.0,
                feature_grad_mult=1.0, extractor_mode=extractor, **NO_DROPOUT)
    torch.manual_seed(4)
    oracle = O.T5TransformerModelASROracle(O.base_asr_args(**over)).train()
    _sharpen(oracle)
    state = TW.round_tree({k: v.clone() for k, v in oracle.state_dict().items()})
    s = O.synthetic_asr_batch(2, 160000, 12, seed=3)
    # utterance 1: one token + eos (CTC sees a one-token target)
    s["target"][1] = PAD
    s["target"][1, 0], s["target"][1, 1] = 7, 2
    s["target_lengths"][1] = 2
    prev = s["net_input"]["prev_output_tokens"]
    prev[1] = PAD
    prev[1, 0], prev[1, 1] = 2, 7
    s = TW.round_tree(s)

    def oracle_run(m):
        dt = next(m.parameters()).dtype
        ni = TW.cast_tree(s["net_input"], dt, cuda)
        ss = dict(s, net_input=ni, target=s["target"].to(cuda), target_lengths=s["target_lengths"].to(cuda))
        got = []
        h = m.register_forward_hook(lambda mod, i, o: got.append(o))
        loss, ce, ctc, _ = O.asr_loss(m, ss, ce_weight=0.5, ctc_weight=0.5, label_smoothing=0.1)
        h.remove()
        loss.backward()
        (logits, _), enc = got[0]
        od = torch.float32 if dt == torch.bfloat16 else torch.float64
        frames = (~enc["encoder_padding_mask"][0]).sum(1)
        return (dict(logits=logits.detach().to(od), ctc=enc["encoder_out_for_ctc"][0].detach().to(od).transpose(0, 1)),
                [loss.detach(), ce.detach(), ctc.detach()], _grads(m), frames)

    arms = []
    for m in TW.twin_and_reference(lambda: O.T5TransformerModelASROracle(O.base_asr_args(**over)).train(), state, cuda):
        arms.append(_oracle_run(m, cuda, oracle_run))
        del m
    T, R = arms
    model = _build(cuda, build_speech_encoder=True, build_text_decoder=True, use_conv_pos=True, use_sinc_pos=True,
                   **over)
    model.load_state_dict(_to_reference_names(state, extractor))
    held = _to_oracle_names(dict(model.named_parameters()))
    assert len([n for n in held if n in state]) > 50
    for n, p in held.items():  # every parameter the oracle has holds the oracle's value
        assert n not in state or torch.equal(p.detach().cpu(), state[n]), n
    got = []
    h = model.register_forward_hook(lambda mod, i, o: got.append(o))
    sample = {"net_input": to_device(s["net_input"], cuda), "target": s["target"].to(cuda),
              "target_lengths": s["target_lengths"].to(cuda), "ntokens": s["ntokens"], "task_name": "s2t"}
    loss, _, log = SpeechT5Criterion(None, label_smoothing=0.1, ce_weight=0.5, ctc_weight=0.5)(model, sample)
    h.remove()
    loss.backward()
    (logits, _), enc = got[0]
    outs = dict(logits=logits.detach().float(), ctc=enc["encoder_out_for_ctc"][0].detach().float().transpose(0, 1))
    P = (outs, [loss.detach(), log["ce_loss"], log["ctc_loss"]], _to_oracle_names(_grads(model)))
    assert torch.equal(R[3].cpu(), (~enc["encoder_padding_mask"][0]).sum(1).cpu())
    tw = TW.Twin(f"s2t {extractor}")
    tw.tensor("text logits", P[0]["logits"], T[0]["logits"], R[0]["logits"], rows=s["target_lengths"])
    tw.tensor("ctc logits", P[0]["ctc"], T[0]["ctc"], R[0]["ctc"], rows=R[3])
    for name, a, b, c in zip(("loss", "ce", "ctc"), P[1], T[1], R[1]):
        tw.scalar(f"loss {name}", float(a), b, c)
    assert tw.grads(P[2], T[2], R[2]) > 40
    assert R[2]["speech_encoder_prenet.feature_extractor.conv_layers.0.0.weight"] is not None
    print("\n" + tw.verdict())
    tw.assert_ok()
