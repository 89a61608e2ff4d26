"""The exact fp8 reference (tests/fp8_exact.py) checked on the CPU: its e4m3 codec against
torch's float8_e4m3fn, its error against the documented bound, and ops.fp8_reference (the
fp32 PyTorch reference the GPU tests also use) against it bit for bit on the edge corpus."""
import numpy as np
import pytest
import torch

import fp8_exact as fe
from infinistore_b200 import _infinistore as native
from infinistore_b200 import ops


@pytest.fixture(scope="module")
def corpus():
    rows = fe.write_corpus()
    q, s = fe.quantise(rows)
    return rows, q, s


def _torch_e4m3(v: np.ndarray) -> np.ndarray:
    t = torch.from_numpy(np.asarray(v, dtype=np.float32)).clamp(-448, 448)
    return t.to(torch.float8_e4m3fn).view(torch.uint8).numpy()


def test_decode_table_matches_torch():
    got = torch.arange(256, dtype=torch.int32).to(torch.uint8).view(torch.float8_e4m3fn)
    want = got.float().double().numpy()
    assert np.array_equal(np.isnan(fe.DECODE), np.isnan(want))
    assert np.array_equal(np.where(np.isnan(want), 0, fe.DECODE), np.nan_to_num(want))
    assert np.array_equal(np.signbit(fe.DECODE[:128]), np.zeros(128, bool))
    assert fe.DECODE[0x7E] == 448.0 and fe.DECODE[1] == 2.0 ** -9 and fe.DECODE[8] == 2.0 ** -6
    assert np.isnan(fe.DECODE[0x7F]) and np.isnan(fe.DECODE[0xFF])


def test_encode_matches_torch_on_every_bf16_pattern():
    v = fe.bf16_to_f64(fe.FINITE)
    assert np.array_equal(fe.encode(v), _torch_e4m3(v))


def test_encode_matches_torch_at_midpoints_saturation_and_zero():
    mids = (fe.POS[:-1] + fe.POS[1:]) / 2.0
    f32 = mids.astype(np.float32)
    assert np.array_equal(f32.astype(np.float64), mids)  # every midpoint is an f32 value
    around = np.concatenate([f32, np.nextafter(f32, np.float32(0)), np.nextafter(f32, np.float32(1e9))])
    sat = np.linspace(448.0, 464.0, 257).astype(np.float32)  # (448, 464] and its edge
    edges = np.array([0.0, 2.0 ** -9, 2.0 ** -10, 7 * 2.0 ** -9, 2.0 ** -6, 15 * 2.0 ** -10,
                      2.0 ** -11, 3 * 2.0 ** -11, 1e-30, 464.0, 480.0, 1e30], np.float32)
    for v in (around, sat, edges):
        v = np.concatenate([v, -v]).astype(np.float64)
        assert np.array_equal(fe.encode(v), _torch_e4m3(v))
    assert fe.encode(np.array([-0.0]))[0] == 0x80 and fe.encode(np.array([0.0]))[0] == 0
    assert fe.encode(np.array([np.nan]))[0] == fe.E4M3_NAN
    assert fe.is_tie(mids).all() and not fe.is_tie(fe.POS).any()


def test_ties_round_to_the_even_code():
    mids = (fe.POS[:-1] + fe.POS[1:]) / 2.0
    codes = fe.encode(mids)
    assert (codes % 2 == 0).all()
    lo = np.arange(126)
    assert np.array_equal(codes, np.where(lo % 2 == 0, lo, lo + 1))


def test_row_of_448_has_scale_one():
    x = fe.bf16_to_f64(np.full((1, 128), 0x43E0, np.uint16))  # 448
    assert fe.row_scales(x)[0] == 1.0


def test_corpus_covers_the_edges(corpus):
    rows, q, s = corpus
    x = fe.bf16_to_f64(rows)
    finite = np.isfinite(x).all(axis=1)
    vals = set(np.unique(rows[finite]).tolist())
    assert set(fe.FINITE.tolist()) <= vals  # every finite bf16 pattern
    amax = np.where(np.isfinite(x), np.abs(np.where(np.isfinite(x), x, 0)), 0).max(axis=1)
    tiny = 448.0 / float(np.finfo(np.float32).max)
    assert ((amax > 0) & (amax < tiny)).any() and (amax < 448.0 * 2.0 ** -126).sum() > 10
    assert (s[finite] == np.float32(2.0 ** -126)).sum() > 10  # rows that take the floor
    pos = np.abs(np.where(np.isfinite(x), x, 0)).argmax(axis=1)
    assert len(set(pos[amax > 0].tolist())) == 128  # the maximum at every position
    ties = fe.is_tie(np.where(np.isfinite(x), x, 0)) & (s[:, None] == 1.0)
    assert ties.sum() >= 2 * 126
    assert (~finite).sum() >= 10 and (np.isnan(x).all(axis=1)).any() and np.isinf(x).all(axis=1).any()


def test_finite_rows_within_the_error_bound(corpus):
    rows, q, s = corpus
    x = fe.bf16_to_f64(rows)
    finite = np.isfinite(x).all(axis=1)
    y = fe.bf16_to_f64(fe.dequantise(q[finite], s[finite]))
    err = np.abs(y - x[finite])
    assert np.isfinite(y).all()
    assert (err <= fe.error_bound(x[finite], s[finite])).all()
    assert (s[finite] >= np.float32(2.0 ** -126)).all()


def test_nonfinite_elements_are_nan_and_leave_their_row_alone(corpus):
    rows, q, s = corpus
    x = fe.bf16_to_f64(rows)
    bad = ~np.isfinite(x)
    assert ((q & 0x7F) == 0x7F)[bad].all()
    assert (q[bad] == fe.E4M3_NAN).all()
    row_bad = bad.any(axis=1)
    y = fe.bf16_to_f64(fe.dequantise(q[row_bad], s[row_bad]))
    ok = ~bad[row_bad]
    assert np.isfinite(y[ok]).all() and np.isnan(y[~ok]).all()
    assert np.isfinite(s).all() and (s > 0).all()


def test_tiny_rows_without_the_floor_would_be_nan():
    """The defect the floor fixes, in f32 arithmetic: max |x| = 1e-37 gives inv = inf."""
    amax = np.float32(1e-37)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        scale = amax * np.float32(1 / 448)
        inv = np.float32(1) / scale
        assert np.isinf(inv) and np.isnan(np.float32(0) * inv)
    x = np.zeros((1, 128))
    x[0, 3] = fe.bf16_to_f64(np.array([fe._bf16_of(1e-37)]))[0]
    q, s = fe.quantise(fe.bf16_rne(x))
    assert s[0] == np.float32(2.0 ** -126) and not ((q & 0x7F) == 0x7F).any()


def test_torch_reference_equals_exact_reference(corpus):
    rows, q, s = corpus
    x = torch.from_numpy(rows.view(np.int16)).view(torch.bfloat16)
    dq, scale, payload = ops.fp8_reference(x)
    assert np.array_equal(scale.numpy().view(np.uint32), s.view(np.uint32))
    assert np.array_equal(payload.view(torch.uint8).numpy().reshape(q.shape), q)
    want = fe.dequantise(q, s)
    got = dq.to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16).reshape(want.shape)
    nan = np.isnan(fe.bf16_to_f64(want))
    assert np.array_equal(np.isnan(fe.bf16_to_f64(got)), nan)
    assert np.array_equal(got[~nan], want[~nan])


def test_dequantise_of_the_read_corpus_against_torch():
    payload, scale = fe.read_corpus()
    y = fe.dequantise(payload, scale)
    v = torch.from_numpy(payload).view(torch.float8_e4m3fn).float()
    t = (v * torch.from_numpy(scale)[:, None]).to(torch.bfloat16)
    got = t.view(torch.int16).numpy().view(np.uint16)
    nan = np.isnan(fe.bf16_to_f64(y))
    assert np.array_equal(np.isnan(fe.bf16_to_f64(got)), nan)
    assert np.array_equal(got[~nan], y[~nan])
    assert np.isinf(fe.bf16_to_f64(y)).any() and nan.any()


def test_plan_fp8_refuses_unaligned_pages():
    for variant in (0, 1, 2):
        assert not native.testing.plan_fp8(n=8, elems=8192, variant=variant, aligned16=False,
                                           sm_count=132)["valid"]
