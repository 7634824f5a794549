"""-m gpu: voice conversion (s2s) on the H100 kernels -- the update against the reference's own run
(tests/golden/ref_vc_tiny.npz) in parity and throughput modes, the captured update against the eager one with dropout
and encoder LayerDrop on, the three synthesis modes against each other and the reference, and a 30 s source."""
import numpy as np
import pytest
import torch

from helpers import rel
from test_vc_cpu import fixture, generate_cases, load_generation_state, mv, vc_args, vc_case

pytestmark = pytest.mark.gpu


def _mode(dtype):
    from speecht5_b200.ops import RT
    RT.dtype = dtype
    RT.manual_seed(1)
    RT.disable_device_seed()
    RT.clear_static()
    RT.invalidate_shadows()
    return RT


def test_update_reproduces_the_reference_run(cuda):
    """Parity mode (hi/lo split GEMMs, fused TTS and guided-attention criterion kernels): loss within 5e-3, every logging
    value within 1e-2, the stored gradients within 1e-2 (the bounds of the other reference pins). Throughput mode (bf16):
    loss within 5e-2, the feat_out gradient within 1e-1."""
    blob = fixture()
    want = blob["loss"]
    _mode(torch.float32)
    _, model, crit, sample = vc_case(cuda, blob)
    loss, n, log = crit(model, sample)
    loss.backward()
    assert n == int(want[5]) and abs(loss.item() - want[0]) < 5e-3 * abs(want[0]), (loss.item(), want)
    for k in [k[4:] for k in blob if k.startswith("log/")]:
        w = float(blob["log/" + k])
        assert abs(float(log[k]) - w) <= 1e-2 * max(1.0, abs(w)), (k, log[k], w)
    params = dict(model.named_parameters())
    for k in mv.GRADS:
        err = rel(params[k].grad, torch.from_numpy(blob["grad/" + k]))
        assert err < 1e-2, (k, err)
    _mode(torch.bfloat16)
    _, model, crit, sample = vc_case(cuda, blob)
    loss, n, log = crit(model, sample)
    loss.backward()
    assert abs(loss.item() - want[0]) < 5e-2 * abs(want[0]), (loss.item(), want)
    k = "speech_decoder_postnet.feat_out.weight"
    assert rel(dict(model.named_parameters())[k].grad, torch.from_numpy(blob["grad/" + k])) < 1e-1
    _mode(torch.bfloat16)


def test_captured_update_replays_equal_the_eager_update(cuda):
    """B200Trainer: four s2s updates replayed from one captured CUDA graph give the losses, logging statistics and
    parameters of the same four updates run eagerly (bf16 with its fp32 residual stream, dropout 0.1 drawn from the
    device seed, encoder LayerDrop 0.5 drawn on the host -- the seed drops a layer in some updates and none in another --
    guided-attention heads read through probs_grad_heads). The captured update runs a dropped layer and discards its
    output, the eager one skips it: both must give the next layer the same input and the same dropout masks."""
    from speecht5_b200.ops import RT
    from speecht5_b200.tasks import SpeechT5Task
    from speecht5_b200.trainer import B200Trainer
    blob = fixture()
    RT.dtype = torch.bfloat16
    results = []
    for graph in (False, True):
        RT.manual_seed(3)
        RT.disable_device_seed()
        RT.clear_static()
        RT.invalidate_shadows()
        np.random.seed(5)
        torch.manual_seed(5)
        _, model, crit, sample = vc_case(cuda, blob)
        for mod in model.modules():
            if hasattr(mod, "dropout_p"):
                mod.dropout_p = 0.1
        model.encoder.encoder_layerdrop = 0.5
        host = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in sample.items() if k != "net_input"}
        host["net_input"] = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in sample["net_input"].items()}
        trainer = B200Trainer(model, crit, SpeechT5Task(vc_args()), use_cuda_graph=graph)
        assert RT.probs_grad_heads == 2
        losses, stats, kept = [], [], []
        for _ in range(4):
            lo, st = trainer.train_step([host])
            losses.append(lo.clone())
            stats.append(st.clone())
            kept.append(tuple(trainer._keep_host[:2].tolist()))
        torch.cuda.synchronize()
        results.append((torch.cat(losses), torch.cat(stats), trainer.fp.flat.clone(), kept))
        assert trainer.graph_misses == (1 if graph else 0)
    (l0, s0, p0, k0), (l1, s1, p1, k1) = results
    assert k0 == k1 and (0.0 in sum(k0, ())) and (1.0, 1.0) in k0, k0
    assert torch.isfinite(l0).all() and torch.allclose(l0, l1, rtol=1e-5, atol=1e-6), (l0, l1)
    assert torch.allclose(s0, s1, rtol=1e-5, atol=1e-6)
    assert rel(p1, p0) < 1e-6


def test_synthesis_modes_agree_and_reproduce_the_reference(cuda):
    """generate_speech(source=...) in parity mode: prefix recomputation, key/value cache and one CUDA graph per step give
    the same frames, and the reference's mel / stop probabilities / attention: the whole default budget, a stop on a
    probability before it, and `threshold` passed."""
    blob = fixture()
    _mode(torch.float32)
    _, model, _, _ = vc_case(cuda, blob)
    model.eval()
    load_generation_state(model, blob)
    runs = [generate_cases(model, blob, cuda, use_cache=m) for m in (False, True, "graph")]
    for name in mv.GEN:
        for k, outs in zip(("mel", "probs", "attn"), zip(*[r[name] for r in runs])):
            want = torch.from_numpy(blob[f"gen/{name}/{k}"])
            for o in outs:
                assert o.shape == want.shape and rel(o, want) < 1e-3, (name, k, rel(o, want))
            assert rel(outs[1], outs[0]) < 1e-4 and rel(outs[2], outs[1]) < 1e-4, name
    _mode(torch.bfloat16)


def test_a_30_second_source_trains_and_converts(cuda):
    """One 30 s source (480 256 samples, 1 500 encoder frames) at Base width in bf16: a captured update with finite
    loss and parameters, then graph-mode synthesis (budget 1 500 x 10 / 2 steps) with finite outputs."""
    from speecht5_b200.criterions import SpeechT5Criterion
    from speecht5_b200.data import synthetic_vc_batch
    from speecht5_b200.models import make_args
    from speecht5_b200.tasks import SpeechT5Task
    from speecht5_b200.trainer import B200Trainer
    RT = _mode(torch.bfloat16)
    RT.enable_device_seed(cuda)
    args = make_args("t5_transformer_base_asr", t5_task="s2s", build_speech_encoder=True, mask_prob=0.0,
                     mask_channel_prob=0.0, max_speech_positions=1876)
    task = SpeechT5Task(args)
    torch.manual_seed(0)
    model = task.build_model(args).to(cuda).train()
    crit = SpeechT5Criterion(task, use_guided_attn_loss=True)
    sample = synthetic_vc_batch(1, 480_256, 1_876, seed=3, pin=True)
    trainer = B200Trainer(model, crit, task)
    lo, _ = trainer.train_step([sample])
    torch.cuda.synchronize()
    assert bool(torch.isfinite(lo).all()) and bool(torch.isfinite(trainer.fp.flat).all())
    model.eval()
    ni = sample["net_input"]
    mel, probs, attn = model.generate_speech(source=ni["source"].to(cuda), padding_mask=ni["padding_mask"].to(cuda),
                                             spkembs=ni["spkembs"].to(cuda), use_cache="graph")
    assert attn.shape[-1] == 1500 and 1 <= mel.shape[0] <= 1500 * 10
    assert bool(torch.isfinite(mel).all()) and bool(torch.isfinite(probs).all()) and bool(torch.isfinite(attn).all())
    RT.clear_static()
    RT.invalidate_shadows()
