"""The comparison rule every parity test applies (harness.n_diff): unorm8 codes exactly, f16 / f32 bit for bit with NaN payloads
included, and two NaNs equal only under nan_equal=True, the hostile-input rule.  A looser rule would weaken every parity test at once."""
import numpy as np

from harness import n_diff


def test_one_unorm8_code_counts():
    ref = np.arange(64, dtype=np.uint8).reshape(8, 8)
    got = ref.copy()
    got[3, 5] += 1
    assert n_diff(got, ref) == 1


def test_one_f32_bit_counts():
    ref = np.linspace(0.1, 7.0, 48, dtype=np.float32).reshape(6, 8)
    got = ref.copy()
    got.view(np.uint32)[2, 7] ^= 1
    assert n_diff(got, ref) == 1


def test_f16_nan_payload_counts_unless_nan_equal():
    ref = np.full((4, 4), 0.5, np.float32)
    ref[1, 2] = np.nan                                            # the canonical NaN, 0x7e00 in f16
    got = ref.astype(np.float16)
    got.view(np.uint16)[1, 2] = 0x7e01                            # another NaN payload
    assert n_diff(got, ref) == 1
    assert n_diff(got, ref, nan_equal=True) == 0


def test_equal_buffers_give_zero():
    ref = np.array([[0.0, -0.0, np.inf], [np.nan, 1e-40, 65504.0]], np.float32)
    assert n_diff(ref.copy(), ref) == 0
    assert n_diff(ref.astype(np.float16), ref) == 0
    assert n_diff(np.full((3, 3), 200, np.uint8), np.full((3, 3), 200, np.uint8)) == 0
