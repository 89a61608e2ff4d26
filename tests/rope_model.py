"""A numpy model of the RoPE shift contract (docs/kernels.md, "RoPE shift contract"): what the
segment movers (csrc/kernels/kv_rope.cu) store and land, from the same (cos, sin) table
``rope_table`` gives the kernels.  float32 products and sums, each rounded on its own (no
FMA), and bf16 round-to-nearest-even done on the bits."""
from __future__ import annotations

import numpy as np

from infinistore_b200.lib import RotaryConfig, rope_table  # noqa: F401  (the shared table)


def bf16_to_f32(bits: np.ndarray) -> np.ndarray:
    """bf16 bit patterns (uint16) widened to float32, exactly."""
    return (np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(np.float32)


def f32_to_bf16(x: np.ndarray) -> np.ndarray:
    """float32 -> bf16 bits, round to nearest even; a NaN becomes a quiet NaN."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32)
    rounded = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    nan = np.isnan(np.asarray(x, dtype=np.float32))
    return np.where(nan, np.uint16(0x7FFF), rounded).astype(np.uint16)


def turn_pairs(a_bits: np.ndarray, b_bits: np.ndarray, c: np.ndarray, s: np.ndarray):
    """One pair per element: (a, b) bf16 bits turned by (c, s), broadcasting over the pairs'
    last axis.  Returns the new (a, b) bits."""
    a, b = bf16_to_f32(a_bits), bf16_to_f32(b_bits)
    c, s = np.float32(c) if np.ndim(c) == 0 else c.astype(np.float32), \
        np.float32(s) if np.ndim(s) == 0 else s.astype(np.float32)
    with np.errstate(all="ignore"):
        x = (a * c).astype(np.float32) - (b * s).astype(np.float32)
        y = (a * s).astype(np.float32) + (b * c).astype(np.float32)
    return f32_to_bf16(x.astype(np.float32)), f32_to_bf16(y.astype(np.float32))


def shift_heads(bits: np.ndarray, c: np.ndarray, s: np.ndarray, head_elems: int,
                rot_offset: int, rot_dim: int, interleaved: bool) -> np.ndarray:
    """A part (bf16 bits, any shape whose size is whole heads) with every head's rotary pairs
    turned by the table.  A table of (1, 0) pairs returns the bits unchanged (the call is
    copied verbatim)."""
    bits = np.asarray(bits, dtype=np.uint16)
    if np.all(c == 1) and np.all(s == 0):
        return bits.copy()
    h = bits.reshape(-1, head_elems).copy()
    rot = h[:, rot_offset:rot_offset + rot_dim]
    half = rot_dim // 2
    if interleaved:
        a, b = rot[:, 0::2], rot[:, 1::2]
    else:
        a, b = rot[:, :half], rot[:, half:]
    a2, b2 = turn_pairs(a, b, c[None, :], s[None, :])
    if interleaved:
        rot[:, 0::2], rot[:, 1::2] = a2, b2
    else:
        rot[:, :half], rot[:, half:] = a2, b2
    h[:, rot_offset:rot_offset + rot_dim] = rot
    return h.reshape(bits.shape)


def shift_parts(parts, rotary: RotaryConfig, shift: int, head_elems: int, rot_offset: int = 0,
                even_parts: bool = False, first_part: int = 0):
    """The movers' output for a list of parts (bf16 bits), stored part first_part + i."""
    c, s = rope_table(rotary, shift)
    out = []
    for i, p in enumerate(parts):
        turns = not even_parts or (first_part + i) % 2 == 0
        out.append(shift_heads(p, c, s, head_elems, rot_offset, rotary.rot_dim,
                               rotary.interleaved) if turns else np.array(p, dtype=np.uint16))
    return out


def edge_corpus() -> np.ndarray:
    """bf16 bit patterns of the edge cases: signed zeros, subnormals, the smallest and largest
    normals, +-Inf, quiet and signalling NaN payloads, ones and a few ordinary values."""
    return np.array([
        0x0000, 0x8000, 0x0001, 0x8001, 0x007F, 0x807F, 0x0080, 0x8080, 0x7F7F, 0xFF7F,
        0x7F80, 0xFF80, 0x7FC0, 0xFFC0, 0x7F81, 0xFF81, 0x7FFF, 0x3F80, 0xBF80, 0x4049,
        0x3C00, 0x447A, 0xC2F7, 0x0100,
    ], dtype=np.uint16)


def same_bits(x: np.ndarray, y: np.ndarray) -> bool:
    """bf16 bits equal, with any NaN equal to any NaN."""
    x, y = np.asarray(x, dtype=np.uint16), np.asarray(y, dtype=np.uint16)
    nx = (x & 0x7FFF) > 0x7F80
    ny = (y & 0x7FFF) > 0x7F80
    return bool(np.array_equal(nx, ny) and np.array_equal(np.where(nx, 0, x), np.where(ny, 0, y)))
