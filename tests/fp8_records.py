"""A numpy model of fp8 token records (``lib.FP8Records``), built on the exact e4m3 reference
of ``fp8_exact``: a record of one token is

    [latent x e4m3][latent / 128 x fp32 scale][rope x bf16, verbatim]

with each 128-element run of the latent quantised as one row of the fp8 row contract."""
import numpy as np

import fp8_exact as fx


def record_bytes(latent: int, rope: int) -> int:
    return latent + 4 * (latent // fx.ROW) + 2 * rope


def encode(tokens: np.ndarray, latent: int, rope: int) -> np.ndarray:
    """bf16 tokens (bits, uint16 (..., latent + rope)) -> records (uint8 (..., record_bytes))."""
    tokens = np.asarray(tokens, dtype=np.uint16)
    lead = tokens.shape[:-1]
    q, scale = fx.quantise(tokens[..., :latent].reshape(*lead, latent // fx.ROW, fx.ROW))
    return np.concatenate([q.reshape(*lead, latent),
                           scale.astype(np.float32).view(np.uint8).reshape(*lead, -1),
                           np.ascontiguousarray(tokens[..., latent:]).view(np.uint8)], axis=-1)


def decode(records: np.ndarray, latent: int, rope: int) -> np.ndarray:
    """Records (uint8 (..., record_bytes)) -> bf16 tokens (bits, uint16 (..., latent + rope)):
    each latent row ``bf16_rne(e4m3 * scale)``, the rope elements as stored."""
    records = np.ascontiguousarray(records, dtype=np.uint8)
    lead, groups = records.shape[:-1], latent // fx.ROW
    q = records[..., :latent].reshape(*lead, groups, fx.ROW)
    scale = np.ascontiguousarray(records[..., latent:latent + 4 * groups]).view(np.float32)
    lat = fx.dequantise(q, scale).reshape(*lead, latent)
    rp = np.ascontiguousarray(records[..., latent + 4 * groups:]).view(np.uint16)
    return np.concatenate([lat, rp], axis=-1).astype(np.uint16)


def corpus_tokens(latent: int, rope: int, seed: int = 7) -> np.ndarray:
    """Tokens (bits, (T, latent + rope)) whose latent rows are ``fp8_exact.write_corpus()`` in
    order, and whose rope elements are random bf16 with NaN (several payloads), +-inf, zeros
    and subnormals mixed in."""
    rows = fx.write_corpus()
    groups = latent // fx.ROW
    t = -(-len(rows) // groups)
    rows = np.concatenate([rows, np.zeros((t * groups - len(rows), fx.ROW), np.uint16)])
    rng = np.random.default_rng(seed)
    rp = fx.bf16_rne(fx.rn32(rng.standard_normal((t, rope)) * 4.0))
    special = np.array([*fx.NAN_PATTERNS, fx.INF, fx.NINF, 0x0000, 0x8000, 0x0001, 0x807F],
                       dtype=np.uint16)
    mask = rng.random((t, rope)) < 0.1
    rp[mask] = special[rng.integers(0, len(special), int(mask.sum()))]
    return np.concatenate([rows.reshape(t, latent), rp], axis=-1).astype(np.uint16)
