"""-m gpu: the convolutions built on st5_gemm_bf16 over overlapping-window operand views -- the post-net Conv1d k5
(ops.conv1d_k5), the strided front-end layers 1-6 (frontend.StridedConvGeluFn), the grouped positional conv
(frontend.GroupedPosConvFn) and the HiFi-GAN convolutions (vocoder._conv_same, _conv_transpose) -- called as the
model calls them, forward and backward, in both numeric modes, against the fp64 statements of tests/conv_ref.py with
ELEMENTWISE bounds. Every buffer the compositions allocate with torch.empty / empty_like starts NaN
(tests/conv_cases.py), so a row, phase or column slice that no GEMM writes fails; input frames that no output window
covers must get an exactly zero gradient. The largest err / bound per composition is printed at the end (run with -s).

Shapes: both post-net widths and T around the 64-row tile (with one bf16 weight gradient split over the batch
dimension with a zero tail and one not split); every (kernel, stride) of the extractor at 32 and 512 channels, T at
every residue mod the stride and T = k, with GELU and without (layer_norm mode), and one 10 s layer-1 input; the
positional conv of Base and Large with T below the kernel width and B = 3 (its weight gradient runs over the
utterances flattened); the HiFi-GAN kernel / dilation grid with T small enough that dilation phases have no rows."""
import pytest
import torch

import conv_cases as CC

pytestmark = pytest.mark.gpu

REPORT = {}
MODES = [torch.bfloat16, torch.float32]
MODE_IDS = ["bf16", "fp32"]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if REPORT:
        print("\nlargest err / bound per composition:")
        for k in sorted(REPORT):
            print(f"  {k:32s} {REPORT[k]:.3g}")


# ------------------------------------------------------------------------------------------------ post-net
@pytest.mark.parametrize("dtype", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("chans", [(80, 256), (256, 256), (256, 80)], ids=["80-256", "256-256", "256-80"])
def test_postnet_conv(cuda, chans, B, dtype):
    Cin, Cout = chans
    for T in (1, 2, 63, 64, 65, 700):
        r, _ = CC.postnet(cuda, Cin, Cout, B, T, dtype, seed=T + B)
        CC.merge(REPORT, r)


def test_postnet_weight_gradient_split_and_unsplit(cuda):
    """bf16: B = 3, T = 700 splits the weight-gradient contraction over the batch dimension (S > 1) with chunks that
    run past the last frame into the zero tail; B = 1 does not split (S = 1, one GEMM over all frames)."""
    r, info = CC.postnet(cuda, 80, 256, 3, 700, torch.bfloat16, seed=5)
    assert info["split"] and info["S"] > 1 and info["S"] * info["chunk"] > info["Kd"], info
    CC.merge(REPORT, r)
    r, info = CC.postnet(cuda, 80, 256, 1, 700, torch.bfloat16, seed=6)
    assert info["S"] == 1 and not info["split"], info
    CC.merge(REPORT, r)


# ------------------------------------------------------------------------------------------------ strided front end
KS = [(3, 2), (2, 2), (5, 3), (4, 2), (2, 3)]


@pytest.mark.parametrize("dtype", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("act", ["gelu", None], ids=["gelu", "layer_norm"])
@pytest.mark.parametrize("C", [32, 512])
@pytest.mark.parametrize("ks", KS, ids=[f"k{k}s{s}" for k, s in KS])
def test_strided_conv(cuda, ks, C, act, dtype):
    """(2, 3): a kernel shorter than the stride, so one input-gradient phase has no taps (J = 0) and is zeroed."""
    k, s = ks
    for T in [k] + [40 + i for i in range(s)]:
        CC.merge(REPORT, CC.strided(cuda, k, s, C, C, 2, T, act, dtype, seed=T))


@pytest.mark.parametrize("dtype", MODES, ids=MODE_IDS)
def test_strided_conv_10s_layer1(cuda, dtype):
    """Layer 1 of the extractor on 10 s of 16 kHz audio (31 999 frames out of layer 0), forward."""
    CC.merge(REPORT, CC.strided(cuda, 3, 2, 512, 512, 1, 31999, "gelu", dtype, seed=7, backward=False))


# ------------------------------------------------------------------------------------------------ positional conv
POS = [(32, 4, 8), (32, 4, 16), (768, 16, 128), (1024, 16, 128)]


@pytest.mark.parametrize("dtype", MODES, ids=MODE_IDS)
@pytest.mark.parametrize("cgk", POS, ids=[f"C{c}G{g}k{k}" for c, g, k in POS])
def test_positional_conv(cuda, cgk, dtype):
    Cc, G, k = cgk
    for T in (1, 19, 64, 65, 500):
        CC.merge(REPORT, CC.posconv(cuda, Cc, G, k, 3, T, dtype, seed=T))


# ------------------------------------------------------------------------------------------------ HiFi-GAN
TS = (1, 2, 4, 37, 100)


@pytest.mark.parametrize("C", [512, 32])
@pytest.mark.parametrize("d", [1, 3, 5])
@pytest.mark.parametrize("k", [3, 7, 11])
def test_hifigan_conv_same(cuda, k, d, C):
    for residual in (False, True):
        for T in TS:
            CC.merge(REPORT, CC.hifi_same(cuda, C, C, k, d, 2, T, slope=0.1, residual=residual, seed=T,
                                          name="same+res" if residual else "same"))


def test_hifigan_conv_pre_and_post(cuda):
    """conv_pre (80 -> 512, k 7, no activation before it, output allocated by the call) and conv_post (32 -> 1, k 7,
    leaky slope 0.01, tanh, fp32 output with N = 1: the per-thread store path)."""
    for T in TS:
        CC.merge(REPORT, CC.hifi_same(cuda, 80, 512, 7, 1, 2, T, out_buffer=False, seed=T, name="conv_pre"))
        CC.merge(REPORT, CC.hifi_same(cuda, 32, 1, 7, 1, 2, T, slope=0.01, act="tanh", out_dtype=torch.float32,
                                      seed=T, name="conv_post"))


@pytest.mark.parametrize("chans", [(512, 256), (64, 32)], ids=["512-256", "64-32"])
def test_hifigan_conv_transpose(cuda, chans):
    for T in TS:
        CC.merge(REPORT, CC.hifi_transpose(cuda, chans[0], chans[1], 2, T, seed=T))
