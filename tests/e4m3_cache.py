"""A numpy model of the e4m3 cache contract (docs/kernels.md, "e4m3 cache contract"), built on
``fp8_exact``'s ``encode`` / ``decode``: the single expected answer of every e4m3 cache test.

An e4m3 cache part is ``elems`` bytes of float8_e4m3fn with one f32 scale ``s_c`` (value
``e4m3(q) * s_c``).  It is stored as the gathered fp8 page of today: ``elems`` payload bytes,
then ``elems / 128`` f32 group scales.
- Write: the payload is the cache's bytes, NaN codes included; every group scale is ``s_c``.
- Read of a stored group (bytes ``q``, scale ``s_g``) into a cache of scale ``s_c``: the bytes
  verbatim when ``s_g`` and ``s_c`` are the same float, else
  ``e4m3_satfinite_rne(rn32(e4m3(q) * min(rn32(s_g / s_c), FLT_MAX)))``.

Exactness: float64 division of two f32 values rounded once to f32 is the correctly rounded f32
quotient (53 >= 2 * 24 + 2), and ``e4m3(q) * r`` has at most 4 + 24 significant bits, so it is
exact in float64 before ``rn32``.
"""
import numpy as np

from fp8_exact import DECODE, ROW, dequantise, encode, rn32

FLT_MAX = float(np.finfo(np.float32).max)


def f32(x) -> np.ndarray:
    return np.asarray(x, dtype=np.float32)


def ratio(s_g, s_c) -> np.ndarray:
    """min(rn32(s_g / s_c), FLT_MAX) as float64 (f32 values)."""
    with np.errstate(over="ignore", under="ignore"):
        r = rn32(f32(s_g).astype(np.float64) / f32(s_c).astype(np.float64))
    return np.fmin(r, FLT_MAX)


def requant(q, s_g, s_c) -> np.ndarray:
    """Groups ``q`` (uint8, (..., 128)) of stored scales ``s_g`` (...) read into a cache of scale
    ``s_c`` (a scalar or (...)): uint8 (..., 128)."""
    q = np.asarray(q, dtype=np.uint8)
    s_g = f32(s_g)
    s_c = np.broadcast_to(f32(s_c), s_g.shape)
    same = s_g.view(np.uint32) == s_c.view(np.uint32)
    with np.errstate(invalid="ignore", over="ignore"):
        v = rn32(DECODE[q] * ratio(s_g, s_c)[..., None])
    return np.where(same[..., None], q, encode(v)).astype(np.uint8)


def write_part(q, s_c) -> np.ndarray:
    """The stored fp8 page (uint8) of one e4m3 part ``q`` (uint8, elems) at scale ``s_c``."""
    q = np.asarray(q, dtype=np.uint8).reshape(-1)
    scales = np.full(len(q) // ROW, s_c, dtype=np.float32)
    return np.concatenate([q, scales.view(np.uint8)])


def split_part(page: np.ndarray, elems: int):
    """A stored fp8 page -> (payload (elems // 128, 128) uint8, scales (elems // 128,) f32)."""
    page = np.asarray(page, dtype=np.uint8).reshape(-1)
    return page[:elems].reshape(-1, ROW), page[elems:elems + 4 * (elems // ROW)].view(np.float32)


def read_part(page: np.ndarray, elems: int, s_c) -> np.ndarray:
    """What an e4m3 cache of scale ``s_c`` reads from a stored fp8 page: uint8 (elems,)."""
    q, s_g = split_part(page, elems)
    return requant(q, s_g, s_c).reshape(-1)


def read_bf16(page: np.ndarray, elems: int) -> np.ndarray:
    """What a bf16 fp8 read gives for a stored fp8 page: bf16 bits (elems,)."""
    q, s_g = split_part(page, elems)
    return dequantise(q, s_g).reshape(-1)


def cache_bf16(q, s_c) -> np.ndarray:
    """The engine's own dequantisation of e4m3 bytes at scale ``s_c``: bf16_rne(rn32(e4m3(q) *
    s_c)), bf16 bits of the same shape."""
    q = np.asarray(q, dtype=np.uint8)
    return dequantise(q.reshape(-1, ROW), np.full(q.size // ROW, s_c, np.float32)).reshape(q.shape)
