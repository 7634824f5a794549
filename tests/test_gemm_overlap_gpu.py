"""-m gpu: the accumulator handoff of st5_gemm_bf16 (csrc/gemm.cu) between the MMA warpgroups and the epilogue
warpgroup, against the fp64 statement of tests/gemm_emulator.py through test_gemm_contract_gpu.run_gemm.

A CTA walks its tiles with the MMA warps one tile ahead of the epilogue: they store tile i's accumulators into shared
memory, start tile i + 1 and wait for the epilogue to release the buffer before storing that one; on the CTA's last tile
they join the epilogue. The cases below make each side the slow one (K = 64: the MMA warps wait for the epilogue every
tile; K = 3072: the epilogue waits for the MMAs), run every epilogue kind over several tiles per CTA, and mix CTAs with
one and two tiles in one launch. Tile counts are quoted for 132 SMs (H100 SXM); the cases stay valid on other counts.

The cost model picks the tile width: N <= 64 always runs 128 x 64 tiles, the wide shapes below run 128 x 128 (more
than one round of 128 x 128 tiles costs less than twice as many 128 x 64 ones)."""
import pytest
import torch

from test_gemm_contract_gpu import run_gemm

pytestmark = pytest.mark.gpu

# (M, N) per tile width
EPILOGUE_BOUND = {"bn64": (140_000, 64), "bn128": (4100, 4096)}  # 1094 / 1056 tiles: 8 per CTA, K = 64
MAINLOOP_BOUND = {"bn64": (33_000, 64), "bn128": (4100, 1024)}   # 258 / 264 tiles: 2 per CTA, K = 3072
THREE_PER_CTA = {"bn64": (50_700, 64), "bn128": (4100, 1536)}    # 397 / 396 tiles: 3 per CTA
ONE_OR_TWO = {"bn64": (23_290, 64), "bn128": (1790, 1664)}       # 182 tiles: 50 CTAs with two, 82 with one
WIDTH_IDS = ["bn64", "bn128"]


@pytest.mark.parametrize("width", WIDTH_IDS)
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_epilogue_bound(cuda, width, out_dtype):
    """One k-block per tile: the epilogue of every tile is longer than the next tile's main loop."""
    M, N = EPILOGUE_BOUND[width]
    run_gemm(M, N, 64, bias="aligned", out_dtype=out_dtype, seed_data=31)


@pytest.mark.parametrize("width", WIDTH_IDS)
def test_mainloop_bound(cuda, width):
    M, N = MAINLOOP_BOUND[width]
    run_gemm(M, N, 3072, a_mn=True, out_dtype=torch.bfloat16, bias="aligned", seed_data=32)


@pytest.mark.parametrize("width", WIDTH_IDS)
def test_gate_epilogue_over_tiles(cuda, width):
    M, N = THREE_PER_CTA[width]
    r = run_gemm(M, N, 200, act="gelu_tanh_gate", c_pre=True, drop_p=0.1, out_dtype=torch.bfloat16, c_ld=N,
                 seed=7, offset=3, seed_data=33)
    assert torch.isfinite(r["got"]).all()


@pytest.mark.parametrize("width", WIDTH_IDS)
def test_dropout_and_pre_over_tiles(cuda, width):
    """Two outputs of one chunk through the same staging block: c_pre, then the activated, dropped value."""
    M, N = THREE_PER_CTA[width]
    run_gemm(M, N, 200, act="gelu", c_pre=True, drop_p=0.25, bias="aligned", out_dtype=torch.bfloat16,
             seed=11, offset=5, seed_data=34)


@pytest.mark.parametrize("width", WIDTH_IDS)
@pytest.mark.parametrize("ag", ["gelu_tanh", "gate"])
def test_residual_and_actgrad_over_tiles(cuda, width, ag):
    M, N = THREE_PER_CTA[width]
    run_gemm(M, N, 200, actgrad_act=ag, residual=True, out_dtype=torch.bfloat16, seed_data=35)


@pytest.mark.parametrize("width", WIDTH_IDS)
def test_accumulate_2_over_tiles(cuda, width):
    """Split-K into one shared fp32 output: three batch entries of K = 64 reduce-added at the L2."""
    M, N = THREE_PER_CTA[width]
    run_gemm(M, N, 64, nb1=3, shared=True, accumulate=2, a_mn=True, b_mn=True, seed_data=36)


@pytest.mark.parametrize("width", WIDTH_IDS)
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_one_and_two_tile_ctas(cuda, width, out_dtype):
    """Some CTAs hand one tile to the epilogue warpgroup before draining their last with all 12 warps, the others
    only drain one tile with 12 warps; accumulate = 1 reads C in the same epilogue."""
    M, N = ONE_OR_TWO[width]
    if out_dtype == torch.float32:
        run_gemm(M, N, 200, accumulate=1, alpha=0.5, bias="offset", residual=True, seed_data=37)
    else:
        run_gemm(M, N, 200, drop_p=0.1, act="relu", residual=True, out_dtype=out_dtype, seed_data=38)
