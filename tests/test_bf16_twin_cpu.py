"""CPU checks of tests/bf16_twin.py, the throughput-mode yardstick: the twin (bf16) and the reference (fp64) hold the
same values, the bf16 rounding is a projection, the twin lands near the reference on a tiny model, and the comparison
e_P <= C e_T + F |R| computes what it states -- per utterance, max-abs, for analytically zero gradients and at the
floor."""
import math

import pytest
import torch

import bf16_twin as TW
from helpers import NO_DROPOUT, TINY, rel


def _tiny_oracle(seed=0):
    from oracle.speecht5_oracle import T5TransformerModelOracle, base_args
    torch.manual_seed(seed)
    return lambda: T5TransformerModelOracle(base_args(**TINY, **NO_DROPOUT, bert_init=True)).train()


def test_twin_and_reference_hold_identical_values():
    make = _tiny_oracle()
    state = TW.round_tree(make().state_dict())
    T, R = TW.twin_and_reference(make, state, "cpu")
    t_sd, r_sd = T.state_dict(), R.state_dict()
    assert t_sd.keys() == r_sd.keys() == state.keys()
    n_float = 0
    for k, v in state.items():
        if v.is_floating_point():
            n_float += 1
            assert t_sd[k].dtype == torch.bfloat16 and r_sd[k].dtype == torch.float64, k
            assert torch.equal(t_sd[k].double(), r_sd[k]) and torch.equal(r_sd[k], v.double()), k
        else:
            assert torch.equal(t_sd[k], v) and torch.equal(r_sd[k], v), k
    assert n_float > 50
    # without the rounding the two arms would not hold the same weights
    raw = make().state_dict()
    T2, R2 = TW.twin_and_reference(make, raw, "cpu")
    k = "encoder.layers.0.fc1.weight"
    assert not torch.equal(T2.state_dict()[k].double(), R2.state_dict()[k])


def test_bf16_rounding_is_idempotent_and_representable():
    g = torch.Generator().manual_seed(1)
    for dtype in (torch.float32, torch.float64):
        x = (torch.randn(4097, generator=g, dtype=torch.float64) * torch.logspace(-20, 20, 4097, dtype=torch.float64)).to(dtype)
        x[:4] = torch.tensor([0.0, -0.0, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8], dtype=dtype)  # ties to even
        y = TW.bf16_exact(x)
        assert y.dtype == dtype
        assert torch.equal(TW.bf16_exact(y), y)
        assert torch.equal(y.to(torch.bfloat16).to(dtype), y)
        nz = x != 0
        assert float(((y - x).double().abs()[nz] / x.double().abs()[nz]).max()) <= 2.0 ** -8  # unit roundoff
        assert y[2] == 1.0 and y[3] == 1.0 + 2.0 ** -6
    batch = {"a": torch.tensor([1, 2, 3]), "m": torch.tensor([True, False]), "s": "t2s",
             "x": [torch.tensor([0.1], dtype=torch.float32)]}
    out = TW.round_tree(batch)
    assert out["a"].dtype == torch.int64 and torch.equal(out["a"], batch["a"]) and torch.equal(out["m"], batch["m"])
    assert out["s"] == "t2s" and out["x"][0].item() == torch.tensor(0.1).bfloat16().float().item()


def test_twin_in_bf16_lands_near_the_fp64_reference_on_a_tiny_model():
    from oracle.speecht5_oracle import synthetic_tts_batch, tts_loss
    make = _tiny_oracle(3)
    state = TW.round_tree(make().state_dict())
    sample = TW.round_tree(synthetic_tts_batch(3, 12, 20, seed=2))
    T, R = TW.twin_and_reference(make, state, "cpu")
    F32 = make()
    F32.load_state_dict(state)
    scales = TW.alpha_scales(R)
    outs = []
    for m, dt in ((T, torch.float32), (R, torch.float64), (F32, torch.float32)):
        ni = TW.cast_tree(sample["net_input"], next(m.parameters()).dtype)
        before, after, logits, attn = m(**ni)
        out = [before.to(dt), after.to(dt), logits.to(dt), [a.to(dt) for a in attn]]
        loss = tts_loss(out, TW.cast_tree(sample, dt))[0]
        loss.backward()
        outs.append((out[1].detach(), float(loss.detach()), TW.param_grads(m)))
    (at, lt, gt), (ar, lr, gr), (af, lf, gf) = outs
    e_t = rel(at, ar)
    assert 1e-4 < e_t < 3e-2, e_t              # bf16: a few 2^-8 after 2 + 2 layers and the post-net
    assert rel(af, ar) < 1e-5                  # fp32 against fp64: R's own floor is far below bf16
    assert abs(lt - lr) / abs(lr) < 3e-2
    worst = max(rel(gt[n], g) for n, g in gr.items() if g is not None and float(g.norm()) > 1e-3)
    assert worst < 0.5, worst
    # an fp32 run in place of P passes the twin check with room to spare
    tw = TW.Twin("cpu fp32 vs twin", report=False)
    tw.tensor("after", af, at, ar, rows=sample["dec_target_lengths"])
    assert sorted(scales) == ["speech_decoder_prenet.decoder_prenet.1.alpha", "text_encoder_prenet.encoder_prenet.1.alpha"]
    assert all(scales[n] >= abs(float(gr[n])) for n in scales)  # sum |terms| bounds the sum
    tw.grads(gf, gt, gr, scalar_abs=scales)
    tw.assert_ok()
    assert tw.worst < 0.5, tw.verdict()


def test_ratio_arithmetic():
    r = torch.ones(100, dtype=torch.float64)
    t = r + 0.01
    F = TW.F_TWIN
    # e_P = 0.02 * 10, C e_T = 0.02 * 10, F |R| = F * 10
    assert TW.ratio(r + 0.02, t, r) == pytest.approx(0.2 / (0.2 + F * 10), rel=1e-12)
    assert TW.ratio(r + 0.02 + 3 * F, t, r) > 1.0
    assert TW.ratio(r - 0.02, t, r) == TW.ratio(r + 0.02, t, r)
    # the floor: T equal to R, P off by F / 2 relative passes, by 2 F fails
    assert TW.ratio(r * (1 + F / 2), r, r) == pytest.approx(0.5, rel=1e-9)
    assert TW.ratio(r * (1 + 2 * F), r, r) == pytest.approx(2.0, rel=1e-9)
    assert TW.ratio(r, r, r) == 0.0
    assert TW.ratio(r, torch.zeros_like(r), torch.zeros_like(r)) == math.inf
    # max-abs: one outlier of P counts in full
    p = r.clone()
    p[17] += 0.05
    assert TW.ratio_max(p, t, r) == pytest.approx(0.05 / (0.02 + F), rel=1e-12)
    assert TW.ratio_max(p, t, r, C=5.0) < 1.0
    # analytically zero: |P| against C |T| + F gmax
    assert TW.ratio_zero(torch.full((4,), 1e-3), torch.full((4,), 1e-3), gmax=1.0) == pytest.approx(
        2e-3 / (2 * 2e-3 + F), rel=1e-6)


def test_twin_collector_per_utterance_rows_zero_gradients_and_missing():
    g = torch.Generator().manual_seed(0)
    r = torch.randn(3, 10, 4, generator=g, dtype=torch.float64)
    t = r + 1e-2 * torch.randn(3, 10, 4, generator=g, dtype=torch.float64)
    p = r + 0.5 * (t - r)
    rows = torch.tensor([10, 6, 1])
    p[1, 6:] = 1e9  # rows past an utterance's length are not compared
    p[2, 1:] = float("nan")
    tw = TW.Twin("synthetic", report=False)
    assert tw.tensor("x", p, t, r, rows=rows) == pytest.approx(0.5 * TW.C_TWIN ** -1, rel=1e-2)
    assert not tw.fails and tw.n == 4
    p[1, 5, 0] += 1.0  # a fault inside utterance 1 fails its row and the max-abs check
    tw = TW.Twin("synthetic", report=False)
    tw.tensor("x", p, t, r, rows=rows)
    assert sorted(w for w, _ in tw.fails) == ["x max-abs", "x[1]"]
    # gradients: one analytically zero (R at the fp64 floor), one missing in P, one with no gradient anywhere
    gr = {"w": torch.ones(8, dtype=torch.float64), "kb": torch.full((8,), 1e-12, dtype=torch.float64),
          "gone": torch.ones(2, dtype=torch.float64), "dead": None}
    gt = {"w": torch.ones(8) * 1.01, "kb": torch.full((8,), 1e-3), "gone": torch.ones(2), "dead": None}
    gp = {"w": torch.ones(8) * 1.015, "kb": torch.full((8,), 1e-3), "dead": None}
    tw = TW.Twin("grads", report=False)
    assert tw.grads(gp, gt, gr) == 2
    assert [w for w, _ in tw.fails] == ["grad gone missing (P)"]
    del gr["gone"], gt["gone"]
    assert tw.worst < 1.0
    gp["kb"] = torch.full((8,), 3e-3)  # 3e-3 > 2 * 1e-3 + F * gmax / sqrt(8) per element
    tw = TW.Twin("grads", report=False)
    tw.grads(gp, gt, gr)
    assert "grad kb (zero)" in [w for w, _ in tw.fails]
    # a scalar gradient needs its a-priori scale sum |terms|; with it, (2)
    gr["a"], gt["a"], gp["a"] = torch.tensor([0.5], dtype=torch.float64), torch.tensor([0.5001]), torch.tensor([0.5])
    gp["kb"] = torch.full((8,), 1e-3)
    tw = TW.Twin("grads", report=False)
    tw.grads(gp, gt, gr)
    assert "grad a: a scalar without an a-priori scale" in [w for w, _ in tw.fails]
    tw = TW.Twin("grads", report=False)
    gp["gone"] = torch.ones(2)
    gp["a"] = torch.tensor([0.5 + 0.03])
    tw.grads(gp, gt, gr, scalar_abs={"a": 8.0})  # 0.03 <= 2 * 1e-4 + 2^-8 * 8 = 0.0315
    assert not tw.fails and tw.worst == pytest.approx(0.03 / (2 * 1e-4 + 8 * TW.U_BF16), rel=1e-3)
    # loss terms: device / host scalars and Python floats mix; the floor is U |R| (non-negative terms)
    tw = TW.Twin("loss", report=False)
    tw.scalar("l", 1.0 + 1e-3, torch.tensor(1.0 + 1e-3, dtype=torch.float64), torch.tensor(1.0, dtype=torch.float64))
    assert tw.worst == pytest.approx(1e-3 / (2e-3 + TW.U_BF16), rel=1e-9)
    tw.scalar("l off by 1 %", 1.01, 1.0 + 1e-4, 1.0)  # a loss normalisation 1 % off fails
    assert [w for w, _ in tw.fails] == ["l off by 1 %"]
