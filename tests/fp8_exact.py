"""An exact reference of the fp8 row contract (docs/kernels.md, "fp8 row contract"), written
in numpy float64 from the e4m3 bit layout: it shares no code and no arithmetic with the
kernels or with torch's float8 dtype, so a mistake in the kernels' f32 formula cannot hide
in it.  Also the edge corpus the fp8 tests run every kernel on.

Exactness:
- A product of two f32 values has at most 48 significant bits, so it is exact in float64;
  rounding it to f32 once (``rn32``) is the f32 product.
- float64 division is correctly rounded, and rounding that quotient to f32 gives the
  correctly rounded f32 quotient, because 53 >= 2 * 24 + 2 (double rounding is innocuous).
- Sums and differences are never formed: round-to-nearest compares ``2 * v`` with
  ``lo + hi`` of two adjacent e4m3 values, both exact in float64.
"""
import numpy as np

E4M3_NAN = 0x7F
E4M3_MAX = 448.0
MIN_SCALE = 2.0 ** -126
ROW = 128


def _decode_table() -> np.ndarray:
    codes = np.arange(256)
    sign = np.where(codes & 0x80, -1.0, 1.0)
    e = (codes >> 3) & 0xF
    m = (codes & 7).astype(np.float64)
    mag = np.where(e == 0, m * 2.0 ** -9, (1.0 + m / 8.0) * np.exp2(e.astype(np.float64) - 7))
    out = sign * mag
    out[(codes & 0x7F) == 0x7F] = np.nan  # S.1111.111: the only NaN, no infinities
    return out


DECODE = _decode_table()  # float64 value of every e4m3 code
POS = DECODE[:127]        # codes 0..126: the non-negative finite values, increasing


def rn32(x) -> np.ndarray:
    """float64 -> nearest f32 (ties to even), as float64."""
    return np.asarray(x, dtype=np.float64).astype(np.float32).astype(np.float64)


def f32_bits(x) -> np.ndarray:
    return np.asarray(x, dtype=np.float64).astype(np.float32).view(np.uint32)


def bf16_to_f64(bits) -> np.ndarray:
    with np.errstate(invalid="ignore"):  # signalling NaN patterns
        return (np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(
            np.float32).astype(np.float64)


def bf16_rne(x) -> np.ndarray:
    """f32 values (given as float64) -> bf16 bits, round to nearest even; NaN stays NaN."""
    u = f32_bits(x).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    nan = np.isnan(np.asarray(x, dtype=np.float64))
    return np.where(nan, np.uint16(0x7FC0) | (r & np.uint16(0x8000)), r).astype(np.uint16)


def encode(v) -> np.ndarray:
    """Values (float64) -> e4m3 codes: nearest finite value, ties to the even code, |v| above
    448 saturates to 448, the sign (of zero too) is copied, NaN -> the NaN code."""
    v = np.asarray(v, dtype=np.float64)
    a = np.abs(v)
    idx = np.clip(np.searchsorted(POS, a, side="right") - 1, 0, 126)  # POS[idx] <= a
    nxt = np.minimum(idx + 1, 126)
    twice, mid = 2.0 * a, POS[idx] + POS[nxt]
    up = (twice > mid) | ((twice == mid) & (idx % 2 == 1))
    code = np.where(up & (idx < 126), nxt, idx)
    code = np.where(a >= E4M3_MAX, 126, code).astype(np.uint8)
    code = code | np.where(np.signbit(v), np.uint8(0x80), np.uint8(0))
    return np.where(np.isnan(v), np.uint8(E4M3_NAN), code).astype(np.uint8)


def is_tie(v) -> np.ndarray:
    """True where |v| lies exactly halfway between two adjacent finite e4m3 values."""
    a = np.abs(np.asarray(v, dtype=np.float64))
    idx = np.clip(np.searchsorted(POS, a, side="right") - 1, 0, 125)
    return (a < E4M3_MAX) & (2.0 * a == POS[idx] + POS[idx + 1])


def row_scales(x: np.ndarray) -> np.ndarray:
    """Rows of f32 values (float64, shape (..., 128)) -> the f32 scale of each row."""
    finite = np.isfinite(x)
    amax = np.where(finite, np.abs(np.where(finite, x, 0.0)), 0.0).max(axis=-1)
    return np.where(amax > 0, np.maximum(rn32(amax * rn32(1.0 / E4M3_MAX)), MIN_SCALE), 1.0)


def quantise(bits: np.ndarray):
    """bf16 rows (bits, shape (..., 128)) -> (payload uint8 (..., 128), scale f32 (...))."""
    x = bf16_to_f64(bits)
    scale = row_scales(x)
    inv = rn32(1.0 / scale)
    with np.errstate(invalid="ignore"):
        scaled = rn32(x * inv[..., None])
    q = np.where(np.isfinite(x), encode(scaled), np.uint8(E4M3_NAN)).astype(np.uint8)
    return q, scale.astype(np.float32)


def dequantise(payload: np.ndarray, scale: np.ndarray) -> np.ndarray:
    """Payload rows (uint8, (..., 128)) and their f32 scales -> bf16 bits."""
    with np.errstate(invalid="ignore", over="ignore"):
        prod = rn32(DECODE[payload] * np.asarray(scale, dtype=np.float64)[..., None])
    return bf16_rne(prod)


def error_bound(x: np.ndarray, scale: np.ndarray) -> np.ndarray:
    """Largest |y - x| the contract allows for finite rows (float64, (..., 128)):
    e4m3 rounding is at most half an ulp, 2^-4 |v| for normal codes and 2^-10 for subnormal
    ones (in units of the scale); rn32 of x * inv and of q * scale adds 2^-24 relative each,
    and inv * scale differs from 1 by at most 2^-24; bf16 rounding adds 2^-9 relative, or
    2^-134 among bf16 subnormals.  Together:
        |y - x| <= 2^-4 (1 + 2^-4) |x| + 2^-10 (1 + 2^-4) scale + 2^-133.
    A row below the floor (max |x| < 448 * 2^-126) has scale 2^-126, so its absolute term is
    2^-136 (1 + 2^-4): finer than half a bf16 subnormal step, 2^-134."""
    s = np.asarray(scale, dtype=np.float64)[..., None]
    return 2.0 ** -4 * (1 + 2.0 ** -4) * np.abs(x) + 2.0 ** -10 * (1 + 2.0 ** -4) * s + 2.0 ** -133


# ---------------------------------------------------------------------------- the corpus
BF16_MAX = 0x7F7F
NAN_PATTERNS = (0x7FC0, 0xFFC0, 0x7F81, 0xFFFF)
INF, NINF = 0x7F80, 0xFF80


def _bf16_of(v: float) -> int:
    return int(bf16_rne(rn32(v)))


def _bf16_below_above(v: float):
    """The bf16 values just below and just above v (positive, not a bf16 value itself)."""
    b = int(f32_bits(v)) >> 16  # truncation: the bf16 below
    return b, b + 1


def row_maxima(rng: np.random.Generator):
    """bf16 bit patterns used as row maxima A."""
    out = {_bf16_of(448.0), BF16_MAX, _bf16_of(2.0 ** -126), 0x0001, 0x0040, 0x007F}
    out |= {_bf16_of(2.0 ** k) for k in range(-133, 128, 6)}
    for edge in (448.0 * 2.0 ** -126, 448.0 / float(np.finfo(np.float32).max)):
        lo, hi = _bf16_below_above(edge)
        out |= {lo - 1, lo, hi, hi + 1}
    # A * rn32(1/448) rounding up and rounding down
    c = rn32(1.0 / E4M3_MAX)
    cand = rng.integers(0x0080, 0x7F7F, 4000).astype(np.uint16)
    a = bf16_to_f64(cand)
    p = a * c
    r = rn32(p)
    out |= set(int(b) for b in cand[r > p][:4]) | set(int(b) for b in cand[r < p][:4])
    return sorted(out)


FINITE = np.array([b for b in range(0x10000) if (b & 0x7F80) != 0x7F80], dtype=np.uint16)


def _rows_beside(amax_bits: int, rng: np.random.Generator, start: int) -> np.ndarray:
    """Every finite bf16 pattern with |v| <= A, 127 per row, A (alternating sign) at a
    position that moves by one per row."""
    a = bf16_to_f64(amax_bits)
    vals = FINITE[np.abs(bf16_to_f64(FINITE)) <= a]
    vals = vals[rng.permutation(len(vals))]
    nrows = (len(vals) + ROW - 2) // (ROW - 1)
    vals = np.resize(vals, nrows * (ROW - 1)).reshape(nrows, ROW - 1)
    rows = np.empty((nrows, ROW), dtype=np.uint16)
    for i in range(nrows):
        pos = (start + i) % ROW
        sign = 0x8000 if (start + i) % 2 else 0
        rows[i] = np.insert(vals[i], pos, amax_bits | sign)
    return rows


def _special_rows(rng: np.random.Generator) -> np.ndarray:
    rows = []
    one = _bf16_of(1.0)
    # the maximum at each of the 128 positions (every lane and element slot of the shuffle)
    for p in range(ROW):
        m = int(rng.integers(-20, 20))
        r = bf16_rne(rn32(rng.uniform(-1, 1, ROW) * 2.0 ** m))
        r[p] = _bf16_of(2.0 ** (m + 1)) | (0x8000 if p % 2 else 0)
        r[(p + 1) % ROW] &= 0x8000  # a zero beside it
        rows.append(r)
    rows.append(np.zeros(ROW, np.uint16))                                    # all +0
    rows.append(np.full(ROW, 0x8000, np.uint16))                             # all -0
    rows.append(np.where(np.arange(ROW) % 3 == 0, 0x8000, 0).astype(np.uint16))  # mixed zeros
    for p, v in ((0, one), (77, 0x0001), (127, 0x8001), (64, BF16_MAX), (31, 0x0080 | 0x8000)):
        r = np.zeros(ROW, np.uint16)                                         # single non-zero
        r[p] = v
        rows.append(r)
    for a in (one, BF16_MAX, 0x0001, _bf16_of(2.0 ** -126)):
        rows.append(np.full(ROW, a, np.uint16))                              # all A
        rows.append(np.full(ROW, a | 0x8000, np.uint16))                     # all -A
        rows.append(np.where(np.arange(ROW) % 2, a | 0x8000, a).astype(np.uint16))  # alternating
    # exact ties with A = 448 (scale 1): every midpoint of adjacent e4m3 values, both signs,
    # and the bf16 values on either side of each
    mids = (POS[:-1] + POS[1:]) / 2.0
    tb = bf16_rne(rn32(mids))
    ties = np.concatenate([tb, tb - 1, tb + 1]).astype(np.uint16)
    ties = np.concatenate([ties, ties | 0x8000])
    a448 = _bf16_of(448.0)
    for t, i in enumerate(range(0, len(ties), ROW - 1)):
        chunk = np.zeros(ROW - 1, np.uint16)
        chunk[:len(ties[i:i + ROW - 1])] = ties[i:i + ROW - 1]
        rows.append(np.insert(chunk, ROW - 1 - t % ROW, a448))
    return np.stack(rows).astype(np.uint16)


def _nonfinite_rows(rng: np.random.Generator) -> np.ndarray:
    rows = []
    base = bf16_rne(rn32(rng.standard_normal((16, ROW)) * 3))
    for i, (pos, pat) in enumerate([(0, 0x7FC0), (5, 0xFFC0), (64, 0x7F81), (127, 0xFFFF),
                                    (3, INF), (100, NINF), (17, INF), (90, NINF)]):
        r = base[i].copy()
        r[pos] = pat
        rows.append(r)
    r = base[8].copy()
    r[[1, 2, 50]] = [INF, 0x7FC0, NINF]                                       # inf with NaN
    rows.append(r)
    rows.append(np.full(ROW, 0x7FC0, np.uint16))                              # all NaN
    rows.append(np.full(ROW, INF, np.uint16))                                 # all inf
    rows.append(np.where(np.arange(ROW) % 2, NINF, INF).astype(np.uint16))    # all +-inf
    rows.append(np.where(np.arange(ROW) % 2, 0x7FC0, INF).astype(np.uint16))  # inf and NaN only
    r = np.zeros(ROW, np.uint16)
    r[[7, 9]] = [INF, 0x0001]                                                 # inf beside a tiny row
    rows.append(r)
    return np.stack(rows).astype(np.uint16)


def write_corpus(seed: int = 2024) -> np.ndarray:
    """bf16 rows (bits, (R, 128)) for the quantising kernels, shuffled."""
    rng = np.random.default_rng(seed)
    parts = [_rows_beside(a, rng, i * 37) for i, a in enumerate(row_maxima(rng))]
    parts += [_special_rows(rng), _nonfinite_rows(rng)]
    rows = np.concatenate(parts)
    return rows[rng.permutation(len(rows))]


def read_scales() -> np.ndarray:
    """f32 scales of the byte-built pool rows."""
    fmax = float(np.finfo(np.float32).max)
    s = [1.0, 2.0 ** -126, 2.0 ** -149, 2.0 ** -140, 2.0 ** -127 * 1.5,
         float(np.array(0x007FFFFF, np.uint32).view(np.float32)),
         fmax, fmax / 448.0 * 1.25, 2.0 ** 120,        # q * scale overflows bf16 (and f32)
         1.0 + 2.0 ** -8, 3.0 * 2.0 ** -9 + 2.0 ** -20,  # bf16 midpoints, and near one
         -1.0, -3.5, 0.0, -0.0, np.inf, np.nan, 448.0 / fmax]
    s += [2.0 ** k for k in range(-130, 128, 9)]
    return rn32(np.array(s))


def read_corpus():
    """(payload uint8 (R, 128), scale f32 (R,)): all 256 codes at every row position, under
    every scale of read_scales()."""
    k = np.arange(256)[:, None]
    j = np.arange(ROW)[None, :]
    codes = ((k + j * 3) % 256).astype(np.uint8)  # row k: code (k + 3j) mod 256 at position j
    scales = read_scales()
    payload = np.tile(codes, (len(scales), 1))
    scale = np.repeat(scales, 256).astype(np.float32)
    return payload, scale
