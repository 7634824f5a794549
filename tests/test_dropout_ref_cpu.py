"""tests/dropout_ref.py, the host statement of the dropout rule the GPU mask tests compare every kernel with: pinned to
the known answer the kernels' own Philox code gives on the host (test_device_math_cpu.py), keep rates, thresholds."""
import numpy as np

import dropout_ref as D


def test_philox_known_answer():
    x, y, z, w = (int(v) for v in D.philox4x32(1, 2, 3))
    assert (x, y, z, w) == (0x15da0e38, 0x90b50218, 0x61766a43, 0x4b911f60)


def test_philox_uses_the_high_words_of_seed_offset_and_counter():
    base = [int(v) for v in D.philox4x32(1, 2, 3)]
    for args in ((1 | 1 << 32, 2, 3), (1, 2 | 1 << 32, 3), (1, 2, 3 | 1 << 32)):
        assert [int(v) for v in D.philox4x32(*args)] != base, args


def test_lanes_are_the_halves_of_the_four_words_in_order():
    x, y, z, w = (int(v) for v in D.philox4x32(9, 4, 5))
    want = [x & 0xFFFF, x >> 16, y & 0xFFFF, y >> 16, z & 0xFFFF, z >> 16, w & 0xFFFF, w >> 16]
    assert [int(v) for v in D.lanes16(9, 4, np.arange(40, 48))] == want


def test_keep_rates():
    idx = np.arange(1 << 20, dtype=np.uint64)
    for p in (0.1, 0.5):
        rate = D.keep_mask(123456789, 77, idx, p).mean()
        # binomial standard deviation at 2^20 draws is <= 5e-4: 6 sigma
        assert abs(rate - (1 - p)) < 3e-3, (p, rate)


def test_drop_threshold_edges():
    assert D.drop_threshold(0.0) == 0 and D.drop_threshold(-0.5) == 0
    assert D.drop_threshold(1 - 2.0 ** -17) == 65535  # 65535.5 truncates to 65535
    assert D.drop_threshold(1 - 2.0 ** -15) == 65534
    assert D.drop_threshold(65535 / 65536) == 65535
    assert D.drop_threshold(1.0) == 65535 and D.drop_threshold(2.0) == 65535
    assert D.drop_threshold(0.1) == 6553 and D.drop_threshold(0.5) == 32768
    assert D.keep_mask(1, 1, np.arange(64), 0.0).all()


def test_attention_index_rounds_the_pitch_up_to_32():
    assert [D.attn_pitch(t) for t in (1, 29, 32, 33, 313, 499, 512)] == [32, 32, 32, 64, 320, 512, 512]
    assert int(D.attn_index(1, 2, 3, 4, H=4, Tq=10, Tk=313)) == ((1 * 4 + 2) * 10 + 3) * 320 + 4
    m = D.attn_keep(5, 6, 0.3, 2, 3, 7, 29)
    assert m.shape == (2, 3, 7, 29)
    assert m[1, 2, 6, 28] == D.keep_mask(5, 6, ((1 * 3 + 2) * 7 + 6) * 32 + 28, 0.3)
