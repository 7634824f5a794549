"""The full-shape launch replay of test_bench_launches_gpu.py flags small faults: its GEMM checker run with
gemm_emulator standing in for the kernel (on the CPU) passes, and fails when the stand-in drops one k-block of one
output tile that the last persistent CTA computes, or writes one element past the logical output. If the sampling rule
stopped covering the last CTA's tiles, the k-block faults would go unnoticed and this test would fail.

The last CTA's tiles are derived here from csrc/gemm.cu's schedule for 128 x 128 tiles (tile = n_blk * tiles_m + m_blk,
CTA c takes tiles c, c + grid, ...), independently of the checker's own rule."""
import pytest
import torch

import gemm_emulator as E
import test_bench_launches_gpu as BL

SMS = 132
# (M, N, K): 16 x 12 tiles over 132 CTAs, the last CTA owning one interior tile; and the decoder FFN of the benchmarked
# update (M = 32 x 313 rows, N = 3072), 79 x 24 tiles, the last CTA owning 14 of them
SHAPES = {"one_tile": (2048, 1536, 256), "ffn": (10016, 3072, 128)}


def _recorded(M, N, KD):
    """A K.gemm call as launch_census.args_of describes it: K-major operands 16-byte aligned, fp32 output at a row pitch
    of N + 8."""
    return dict(M=M, N=N, K=KD, a_mn=False, b_mn=False, a_ld=None, b_ld=None, c_ld=N + 8, nb1=1, nb2=1, a_bs=(0, 0),
                b_bs=(0, 0), c_bs=(0, 0), bias=None, bias2=None, bias2_rows=0, residual=None, c_pre=None, act=None,
                alpha=1.0, accumulate=False, drop_p=0.0, seed="host", actgrad_pre=None, actgrad_act=None,
                a=("T", "bfloat16", (M, KD), (KD, 1), 0, 0, 0), b=("T", "bfloat16", (N, KD), (KD, 1), 0, 1, 0),
                out=("T", "float32", (M, N), (N + 8, 1), 0, 2, 0))


def _last_cta_tiles(M, N):
    tiles_m, tiles_n = -(-M // 128), -(-N // 128)
    total = tiles_m * tiles_n
    grid = min(total, SMS)
    return [(t % tiles_m * 128, t // tiles_m * 128) for t in range(grid - 1, total, grid)]


def _install(monkeypatch, M, N, fault=None, tile=None):
    from speecht5_b200 import kernels as K

    def gemm(a, b, out, **kw):
        E.gemm(a, b, out, **kw)
        c_ld = kw["c_ld"]
        C = torch.as_strided(out, (M, N), (c_ld, 1), out.storage_offset())
        if fault == "k_block":  # one tile without its first k-block
            m0, n0 = tile
            rows, cols = torch.arange(m0, min(m0 + 128, M)), torch.arange(n0, min(n0 + 128, N))
            part = torch.zeros_like(out)
            E.gemm(a, b, part, **dict(kw, K=64, a_ld=kw["K"], b_ld=kw["K"]), rows=rows, cols=cols)
            P = torch.as_strided(part, (M, N), (c_ld, 1), part.storage_offset())
            C[m0:m0 + 128, n0:n0 + 128] -= P[m0:m0 + 128, n0:n0 + 128]
        elif fault == "past_end":  # one element in the row padding [N, c_ld) of the last row
            torch.as_strided(out, (M, c_ld), (c_ld, 1), out.storage_offset())[M - 1, N] = 0.0
        return out
    monkeypatch.setattr(K, "gemm", gemm)


def test_last_cta_tiles_are_sampled():
    for M, N, _ in SHAPES.values():
        tiles = _last_cta_tiles(M, N)
        blocks = {(int(r[0]), int(c[0])) for r, c in BL.gemm_blocks(M, N, 1, SMS)
                  if r is not None and c is not None and len(c) == 128}
        assert set(tiles) <= blocks
    assert len(_last_cta_tiles(*SHAPES["ffn"][:2])) == 14


def test_unmodified_emulator_passes(monkeypatch):
    M, N, KD = SHAPES["one_tile"]
    _install(monkeypatch, M, N)
    assert BL.replay_gemm(_recorded(M, N, KD), SMS, dev="cpu") <= 1.0


@pytest.mark.parametrize("shape,which", [("one_tile", -1), ("ffn", 6), ("ffn", -1)],
                         ids=["one_tile-last", "ffn-seventh", "ffn-last"])
def test_missing_k_block_in_a_last_cta_tile_is_flagged(monkeypatch, shape, which):
    """The seventh of the FFN's 14 tiles is interior (no first / last 128 rows or columns): only the last-CTA rule
    covers it."""
    M, N, KD = SHAPES[shape]
    m0, n0 = _last_cta_tiles(M, N)[which]
    if which == 6:
        assert 0 < m0 < M - 128 and 0 < n0 < N - 128
    _install(monkeypatch, M, N, "k_block", (m0, n0))
    with pytest.raises(AssertionError, match=rf"first \(b2, b1, m, n\) = \(0, 0, {m0}, {n0}\)"):
        BL.replay_gemm(_recorded(M, N, KD), SMS, dev="cpu")


def test_write_past_the_output_is_flagged(monkeypatch):
    M, N, KD = SHAPES["one_tile"]
    _install(monkeypatch, M, N, "past_end")
    with pytest.raises(AssertionError, match="written outside"):
        BL.replay_gemm(_recorded(M, N, KD), SMS, dev="cpu")
