"""CPU: the e4m3 rule of compute_type="float8_float16" as the oracle states it (oracle/fp8_oracle.py), checked against an
e4m3 grid decoded here from the bit patterns: every finite code maps to itself, midpoints between neighbours round to the
even code, values beyond 448 saturate, and rows of zeros get scale 1 and zero codes."""
import numpy as np
import pytest
import torch

from oracle import fp8_oracle as f8


def e4m3_value(byte: int) -> float:
    """OCP e4m3 (e4m3fn): 1 sign, 4 exponent (bias 7), 3 mantissa bits; S.1111.111 is NaN, there are no infinities."""
    s, e, m = byte >> 7, (byte >> 3) & 15, byte & 7
    if e == 15 and m == 7:
        return float("nan")
    v = (m / 8.0) * 2.0 ** -6 if e == 0 else (1 + m / 8.0) * 2.0 ** (e - 7)
    return -v if s else v


FINITE = [(b, e4m3_value(b)) for b in range(256) if not np.isnan(e4m3_value(b))]
POSITIVE = sorted((v, b) for b, v in FINITE if b < 128)  # +0 .. 448, byte order == value order


def as_bytes(x: np.ndarray) -> np.ndarray:
    return f8.round_e4m3(torch.from_numpy(np.asarray(x, np.float32))).view(torch.uint8).numpy()


def test_grid_is_the_e4m3_grid():
    assert len(FINITE) == 254 and POSITIVE[-1] == (448.0, 0x7E) and POSITIVE[1][0] == 2.0 ** -9


def test_every_finite_code_maps_to_itself():
    bytes_ = np.array([b for b, _ in FINITE], np.uint8)
    vals = np.array([v for _, v in FINITE], np.float32)
    assert (as_bytes(vals) == bytes_).all()


def test_midpoints_round_to_even_code():
    for sign in (1.0, -1.0):
        lo, hi = np.array(POSITIVE[:-1]), np.array(POSITIVE[1:])
        mid = (lo[:, 0] + hi[:, 0]) / 2  # exact in float32: adjacent e4m3 values differ in one bit below 4 significant bits
        assert (mid.astype(np.float32) == mid).all()
        want = np.where(lo[:, 1].astype(int) % 2 == 0, lo[:, 1], hi[:, 1]).astype(np.uint8)
        if sign < 0:
            want = want | 0x80
        assert (as_bytes(sign * mid) == want).all()
        # just off the midpoint goes to the nearer neighbour
        nudge = np.nextafter(mid.astype(np.float32), np.float32(np.inf))
        assert (as_bytes(sign * nudge) == (hi[:, 1].astype(np.uint8) | (0x80 if sign < 0 else 0))).all()


def test_saturation_above_448():
    x = np.array([448.0, 449.0, 463.9, 464.0, 480.0, 1e4, 3e38], np.float32)
    assert (as_bytes(x) == 0x7E).all() and (as_bytes(-x) == 0xFE).all()


def test_row_rule():
    rng = np.random.default_rng(0)
    x = rng.standard_normal((6, 192)).astype(np.float32) * np.float32([[1e-3], [1], [7], [300], [1e5], [1]])
    x[5] = 0
    q, s = f8.quantize_rows(torch.from_numpy(x))
    amax = np.abs(x).max(1)
    want_s = np.where(amax > 0, amax / np.float32(448), np.float32(1)).astype(np.float32)
    assert (s.numpy() == want_s).all()
    assert (q.view(torch.uint8).numpy()[5] == 0).all() and s[5] == 1.0
    # the row's largest element maps to +-448 exactly; every code is x / s rounded to the grid
    got = q.float().numpy()
    assert (np.abs(got[:5]).max(1) == 448).all()
    grid = np.array(sorted({v for _, v in FINITE}), np.float64)
    r = (x / want_s[:, None]).astype(np.float32).astype(np.float64)
    nearest = grid[np.abs(r[..., None] - grid).argmin(-1)]
    assert (np.abs(got - r) <= np.abs(nearest - r)).all()


def test_zero_row_gets_unit_scale():
    q, s = f8.quantize_rows(torch.zeros(3, 64))
    assert (s == 1).all() and (q.view(torch.uint8) == 0).all()


@pytest.mark.parametrize("K", [64, 320])
def test_fp8_linear_is_the_scaled_code_product(K):
    rng = np.random.default_rng(K)
    a = torch.from_numpy(rng.standard_normal((5, K)).astype(np.float32))
    w = torch.from_numpy(rng.standard_normal((7, K)).astype(np.float32))
    qa, sa = f8.quantize_rows(a)
    qw, sw = f8.quantize_rows(w)
    want = (qa.double().numpy() @ qw.double().numpy().T) * sa.double().numpy()[:, None] * sw.double().numpy()[None]
    assert np.allclose(f8.fp8_linear(qa, sa, qw, sw, None).numpy(), want.astype(np.float32), rtol=0, atol=0)
    # the quantised product is a coarse version of the float32 one
    assert np.abs(want - (a @ w.T).numpy()).max() < 0.1 * np.abs((a @ w.T).numpy()).max()
