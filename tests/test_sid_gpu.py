"""-m gpu: speaker identification (s2c) on the H100 kernels -- csrc/speaker_head.cu against torch fp64 autograd, the
product update against the reference's own run (tests/golden/ref_sid_tiny.npz) in parity and throughput modes, the
captured update against the eager one, and generate_class on one 160 s utterance."""
import pytest
import torch

from helpers import rel
from test_sid_cpu import CASES, fixture, head_state, sid_args, sid_case

pytestmark = pytest.mark.gpu


def _margin_ref(x, target, kind, m, s, easy):
    from oracle.speaker_oracle import margin
    return x if kind == "softmax" else margin(x, target, kind, m, s, easy)


@pytest.mark.parametrize("kind,easy", [("softmax", False), ("amsoftmax", False), ("aamsoftmax", False),
                                       ("aamsoftmax", True)])
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("B", [1, 8, 33])
@pytest.mark.parametrize("N", [5, 1251, 1255])
def test_margin_ce_kernel_matches_fp64_autograd(cuda, kind, easy, eps, B, N):
    """st5_margin_ce_fwd / _bwd, fused (margin + CE in one launch) and as the model and criterion issue them (margin
    logits, then plain CE), against the reference's margin formulas and label-smoothed CE in fp64 autograd. Rows on both
    sides of th = cos(pi - m) and of 0; an ignored (padding) row when B > 1."""
    from oracle.speaker_oracle import label_smoothed_ce
    from speecht5_b200 import _lib, kernels as K
    g = torch.Generator().manual_seed(B * 10007 + N)
    m, s = 0.2, 30.0
    cos = ((torch.rand(B, N, generator=g, dtype=torch.float64) * 2 - 1) * 0.9).float().double()
    target = torch.randint(0, N, (B,), generator=g)
    cos[0, target[0]] = -0.995
    if B > 1:
        cos[1, target[1]] = -0.5
        target[B - 1] = 1  # ignored
    x = cos.clone().requires_grad_()
    z = _margin_ref(x, target, kind, m, s, easy)
    loss, nll, correct, total = label_smoothed_ce(z, target, eps, ignore_index=1)
    (1.3 * loss + 0.7 * nll).backward()
    mode = {"softmax": None, "amsoftmax": (_lib.MARGIN_AM, s, m, 0), "aamsoftmax": (_lib.MARGIN_AAM, s, m, int(easy))}[kind]
    xd, td = cos.float().to(cuda), target.to(cuda)
    mt = None if mode is None else td
    gstat = torch.tensor([1.3, 0.7], device=cuda)
    stats, lse = torch.empty(B, 4, device=cuda), torch.empty(B, device=cuda)
    zk = torch.empty(B, N, device=cuda)
    K.margin_ce_fwd(xd, mt, mode, z_out=zk, target=td, eps=eps, ignore_index=1, stats=stats, lse=lse)
    assert rel(zk, z) < 1e-6
    st = stats.double().sum(0).cpu()
    assert abs(st[0].item() - loss.item()) <= 1e-5 * abs(loss.item()) + 1e-6
    assert abs(st[1].item() - nll.item()) <= 1e-5 * abs(nll.item()) + 1e-6
    assert (int(st[2]), int(st[3])) == (correct, total)
    dx = torch.empty(B, N, device=cuda)
    K.margin_ce_bwd(xd, mt, mode, dx, target=td, eps=eps, ignore_index=1, lse=lse, gstat=gstat)
    assert rel(dx, x.grad) < 1e-5
    # the two halves
    z2 = torch.empty(B, N, device=cuda)
    K.margin_ce_fwd(xd, mt, mode, z_out=z2) if mode is not None else z2.copy_(xd)
    K.margin_ce_fwd(z2, None, None, target=td, eps=eps, ignore_index=1, stats=stats, lse=lse)
    dz, dx2 = torch.empty(B, N, device=cuda), torch.empty(B, N, device=cuda)
    K.margin_ce_bwd(z2, None, None, dz, target=td, eps=eps, ignore_index=1, lse=lse, gstat=gstat)
    K.margin_ce_bwd(xd, mt, mode, dx2, dz=dz)
    assert rel(dx2, x.grad) < 1e-5


@pytest.mark.parametrize("rows,E,dtype", [(1, 64, torch.float32), (8, 768, torch.bfloat16), (1255, 128, torch.float32),
                                          (33, 100, torch.float32)])
def test_l2norm_and_time_mean_kernels_match_fp64_autograd(cuda, rows, E, dtype):
    from speecht5_b200 import kernels as K
    g = torch.Generator().manual_seed(rows + E)
    x = torch.randn(rows, E, generator=g, dtype=torch.float64)
    x[0] *= 1e-14  # a clamped row (norm below 1e-12)
    x = x.to(dtype).double()
    xr = x.clone().requires_grad_()
    y = torch.nn.functional.normalize(xr, p=2, dim=1)
    dy = torch.randn(rows, E, generator=g, dtype=torch.float64)
    (y * dy).sum().backward()
    yk, nk = torch.empty(rows, E, device=cuda), torch.empty(rows, device=cuda)
    K.l2norm_rows_fwd(x.to(dtype).to(cuda), yk, nk)
    assert rel(yk, y) < 1e-6
    dx = torch.empty(rows, E, dtype=dtype, device=cuda)
    K.l2norm_rows_bwd(dy.float().to(cuda), yk, nk, dx)
    assert rel(dx[1:], xr.grad[1:]) < (1e-5 if dtype == torch.float32 else 1e-2)
    assert rel(dx[:1], xr.grad[:1]) < (1e-5 if dtype == torch.float32 else 1e-2)
    acc = torch.ones(rows, E, device=cuda)
    K.l2norm_rows_bwd(dy.float().to(cuda), yk, nk, acc, accumulate=True)
    assert rel(acc - 1.0, xr.grad) < 1e-5 if dtype == torch.float32 else True
    # mean over all frames of [B, T, C]
    xt = torch.randn(3, rows, E, generator=g).to(dtype)
    ym = torch.empty(3, E, dtype=dtype, device=cuda)
    K.time_mean_fwd(xt.to(cuda), ym)
    assert rel(ym, xt.double().mean(1)) < (1e-6 if dtype == torch.float32 else 1e-2)
    dxt = torch.empty(3, rows, E, dtype=dtype, device=cuda)
    K.time_mean_bwd(ym, dxt)
    assert rel(dxt, ym.double().cpu()[:, None, :].expand(3, rows, E) / rows) < 1e-6 if dtype == torch.float32 else True


def _run_case(cuda, name, dtype, blob):
    from speecht5_b200.ops import RT
    RT.dtype = dtype
    RT.manual_seed(1)
    RT.disable_device_seed()
    RT.clear_static()
    RT.invalidate_shadows()
    _, model, crit, sample = sid_case(name, cuda, blob)
    seen = {}
    model.speaker_decoder_postnet.register_forward_hook(lambda m, a, out: seen.__setitem__("out", out))
    loss, n, log = crit(model, sample)
    loss.backward()
    return model, sample, loss, n, log, seen["out"]


@pytest.mark.parametrize("name", CASES)
def test_update_reproduces_the_reference_run(cuda, name):
    """Parity mode (hi/lo split GEMMs): loss, logging values, logits and gradients within the bounds of the other
    reference pins (loss 5e-3, logging 1e-2, gradients 1e-2) and generate_class's predictions exactly. Throughput mode
    (bf16 activations and operands): loss and logits within 5e-2, the head-weight gradient within 1e-1."""
    blob = fixture()
    want = blob[f"{name}/loss"]
    model, sample, loss, n, log, out = _run_case(cuda, name, torch.float32, blob)
    assert n == int(want[4]) and log["ntokens"] == int(want[5])
    assert abs(loss.item() - want[0]) < 5e-3 * abs(want[0]), (loss.item(), want)
    assert abs(log["nll_loss"] - want[1]) < 1e-2 * abs(want[1])
    assert (log["n_correct"], log["total"]) == (int(want[2]), int(want[3]))
    assert rel(out[0], torch.from_numpy(blob[f"{name}/out/logits"])) < 5e-3
    params = dict(model.named_parameters())
    grads = [k[len(name) + 6:] for k in blob if k.startswith(name + "/grad/")]
    assert len(grads) >= 6
    for k in grads:
        err = rel(params[k].grad, torch.from_numpy(blob[f"{name}/grad/{k}"]))
        assert err < 1e-2, (k, err)
    model.load_state_dict(head_state(blob, name), strict=False)  # BatchNorm statistics of the reference's eval
    model.eval()
    ni = sample["net_input"]
    pred = model.generate_class(ni["source"], ni["prev_output_tokens"], padding_mask=ni["padding_mask"])
    assert pred.tolist() == blob[f"{name}/out/pred"].tolist()
    model, sample, loss, n, log, out = _run_case(cuda, name, torch.bfloat16, blob)
    assert abs(loss.item() - want[0]) < 5e-2 * abs(want[0]), (loss.item(), want)
    assert rel(out[0], torch.from_numpy(blob[f"{name}/out/logits"])) < 5e-2
    k = "speaker_decoder_postnet.output_projection.weight"
    assert rel(dict(model.named_parameters())[k].grad, torch.from_numpy(blob[f"{name}/grad/{k}"])) < 1e-1
    from speecht5_b200.ops import RT
    RT.dtype = torch.bfloat16
    RT.clear_static()
    RT.invalidate_shadows()


@pytest.mark.parametrize("name", ["defaults", "aam"])
def test_captured_update_replays_equal_the_eager_update(cuda, name):
    """B200Trainer: three s2c updates replayed from one captured CUDA graph give the losses, logging statistics and
    parameters of the same three updates run eagerly (bf16 throughput mode, dropout 0.1 drawn from the device seed)."""
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
        _, model, crit, sample = sid_case(name, cuda, blob)
        for mod in model.modules():
            if hasattr(mod, "dropout_p"):
                mod.dropout_p = 0.1
        host = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in sample.items() if k != "net_input"}
        host["net_input"] = {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in sample["net_input"].items()}
        trainer = B200Trainer(model, crit, SpeechT5Task(sid_args(name)), use_cuda_graph=graph)
        losses, stats = [], []
        for _ in range(3):
            lo, st = trainer.train_step([host])
            losses.append(lo.clone())
            stats.append(st.clone())
        torch.cuda.synchronize()
        results.append((torch.cat(losses), torch.cat(stats), trainer.fp.flat.clone()))
        assert trainer.graph_misses == (1 if graph else 0)
    (l0, s0, p0), (l1, s1, p1) = results
    assert torch.allclose(l0, l1, rtol=1e-5, atol=1e-6), (l0, l1)
    assert torch.allclose(s0, s1, rtol=1e-5, atol=1e-6)
    assert s0.shape[-1] == 6 and bool((s0[:, 5] == 4).all())  # (loss, ce, ctc, nll, n_correct, total)
    assert rel(p1, p0) < 1e-6


def test_generate_class_on_a_160_second_utterance(cuda):
    """One 160 s utterance (2 560 000 samples, 7 999 encoder frames) through generate_class in bf16 on a reduced-width
    model: the class the parity-mode pooled decoder state gives through the oracle head, no attention probability
    saved for a backward pass, peak memory under 4 GiB."""
    from oracle.speaker_oracle import speaker_head
    from speecht5_b200 import kernels as K
    from speecht5_b200.ops import RT
    from speecht5_b200.tasks import SpeechT5Task
    args = sid_args("recipe", max_speech_positions=8000, conv_feature_layers="[(512, 10, 5)] + [(512, 3, 2)] * 4 + [(512, 2, 2)] * 2")
    torch.manual_seed(5)
    RT.clear_static()
    RT.invalidate_shadows()
    model = SpeechT5Task(args).build_model(args).to(cuda).eval()
    g = torch.Generator().manual_seed(9)
    source = (torch.randn(1, 2_560_000, generator=g) * 0.1).to(cuda)
    pm = torch.zeros_like(source, dtype=torch.bool)
    prev = torch.full((1, 1), 2, dtype=torch.long, device=cuda)
    RT.dtype = torch.float32
    pooled = {}
    h = model.speaker_decoder_postnet.register_forward_pre_hook(lambda m, a: pooled.__setitem__("x", a[0].detach()))
    model.generate_class(source, prev, padding_mask=pm)
    h.remove()
    with torch.no_grad():  # make one class decisive: its weight row along the pooled state
        w = model.speaker_decoder_postnet.output_projection.weight
        w[37] = pooled["x"][0] / pooled["x"][0].norm() * 4.0 * w.norm(dim=1).max()
    RT.invalidate_shadows()
    state = {k: v.detach().cpu() for k, v in model.state_dict().items()}
    ref_logits, _ = speaker_head(state, pooled["x"].cpu(), softmax_type="softmax", pooling_bn=False,
                                 embed_postnet=False, training=False)
    want = int(ref_logits.argmax(1))
    RT.dtype = torch.bfloat16
    RT.invalidate_shadows()
    saved = []
    orig = {n: getattr(K, n) for n in ("attn_flash_fwd", "attn_fused_fwd")}

    def spy(fn):
        def call(a, lse, psave=None, inv_l=None, out_f32=None):
            saved.append(psave is not None or inv_l is not None or out_f32 is not None)
            return fn(a, lse, psave, inv_l, out_f32)
        return call
    for n, fn in orig.items():
        setattr(K, n, spy(fn))
    try:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        pred = model.generate_class(source, prev, padding_mask=pm)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
    finally:
        for n, fn in orig.items():
            setattr(K, n, fn)
    assert int(pred) == want == 37
    assert saved and not any(saved)
    assert peak < 4 * 2 ** 30, peak / 2 ** 30
    RT.clear_static()
    RT.invalidate_shadows()
