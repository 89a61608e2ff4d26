"""Page geometry and key naming for paged KV caches."""
from __future__ import annotations

import hashlib
from dataclasses import dataclass
from typing import Dict, List, Sequence, Tuple

import torch


@dataclass(frozen=True)
class KVLayout:
    """One K (or V) page of one layer = page_tokens x kv_heads x head_dim elements."""

    name: str
    layers: int
    kv_heads: int
    head_dim: int
    page_tokens: int = 128
    dtype: torch.dtype = torch.bfloat16
    tp: int = 1  # tensor-parallel degree: kv heads are split across TP ranks

    @property
    def heads_per_rank(self) -> int:
        return max(self.kv_heads // self.tp, 1)

    @property
    def page_elems(self) -> int:
        return self.page_tokens * self.heads_per_rank * self.head_dim

    @property
    def page_bytes(self) -> int:
        return self.page_elems * torch.empty((), dtype=self.dtype).element_size()

    @property
    def token_bytes_all_layers(self) -> int:
        """K+V bytes one token occupies across all layers on one TP rank."""
        return 2 * self.layers * self.page_bytes // self.page_tokens

    def with_tp(self, tp: int) -> "KVLayout":
        return KVLayout(self.name, self.layers, self.kv_heads, self.head_dim, self.page_tokens,
                        self.dtype, tp)


# GQA configurations of common open models (layers, kv heads, head dim).
LAYOUTS: Dict[str, KVLayout] = {
    "llama-3-8b": KVLayout("llama-3-8b", 32, 8, 128),      # 256 KiB per K or V page per layer
    "llama-3-70b": KVLayout("llama-3-70b", 80, 8, 128),
    "llama-3.1-405b": KVLayout("llama-3.1-405b", 126, 8, 128),
    "mistral-7b": KVLayout("mistral-7b", 32, 8, 128),
    "mixtral-8x7b": KVLayout("mixtral-8x7b", 32, 8, 128),
    "qwen2.5-7b": KVLayout("qwen2.5-7b", 28, 4, 128),
    "qwen2.5-72b": KVLayout("qwen2.5-72b", 80, 8, 128),
    "gemma-2-9b": KVLayout("gemma-2-9b", 42, 8, 256),
    "deepseek-v2-lite-mla": KVLayout("deepseek-v2-lite-mla", 27, 1, 576),  # MLA latent + rope
    "gpt2-xl-mha": KVLayout("gpt2-xl-mha", 48, 25, 64),
}


def get_layout(name: str, page_tokens: int = 128, dtype: torch.dtype = torch.bfloat16,
               tp: int = 1) -> KVLayout:
    base = LAYOUTS[name]
    return KVLayout(base.name, base.layers, base.kv_heads, base.head_dim, page_tokens, dtype, tp)


def chain_hashes(token_ids: Sequence[int], page_tokens: int, salt: str = "") -> List[str]:
    """Prefix-chained page hashes: hash[i] covers tokens [0, (i+1)*page_tokens), so presence
    is prefix-monotone and ``get_match_last_index`` finds the longest cached prefix."""
    out, h = [], hashlib.sha256(salt.encode())
    full = len(token_ids) // page_tokens
    for p in range(full):
        chunk = token_ids[p * page_tokens:(p + 1) * page_tokens]
        h.update(b"".join(int(t).to_bytes(4, "little", signed=False) for t in chunk))
        out.append(h.copy().hexdigest()[:32])
    return out


ALL_LAYERS = "all"  # layer field of a key whose block holds one page of every layer


def _rank_heads(kv_heads: int, tp: int, rank: int) -> List[int]:
    """The KV heads TP rank ``rank`` of ``tp`` holds: ``kv_heads // tp`` consecutive heads, or,
    when ``tp > kv_heads`` (GQA replication), the one head ``rank * kv_heads // tp``."""
    if tp < 1 or (kv_heads % tp and tp % kv_heads):
        raise ValueError(f"TP {tp} neither divides nor is a multiple of {kv_heads} KV heads")
    if not 0 <= rank < tp:
        raise ValueError(f"TP rank {rank} is outside 0..{tp - 1}")
    if tp >= kv_heads:
        return [rank * kv_heads // tp]
    per = kv_heads // tp
    return list(range(rank * per, (rank + 1) * per))


def tp_sources(layout: KVLayout, reader_tp: int, reader_rank: int,
               writer_tp: int) -> List[Tuple[int, int, int, int]]:
    """Where reader rank ``reader_rank`` (of ``reader_tp``) finds its KV heads in pages that
    ranks at ``writer_tp`` wrote: a list of ``(writer_rank, src_head, dst_head, heads)``, each
    ``heads`` consecutive heads from head ``src_head`` of that writer's page to head
    ``dst_head`` of the reader's, in ``dst_head`` order and with equal ``heads``.  A replicated
    head (``tp > kv_heads``) is taken from its first replica.  One source per page when the
    reader holds no more heads than a writer rank (``reader_tp >= writer_tp``, and MLA's single
    latent head), several otherwise.  Raises ``ValueError`` unless both degrees divide, or are
    multiples of, ``layout.kv_heads``."""
    h = layout.kv_heads
    _rank_heads(h, writer_tp, 0)  # checks writer_tp
    out: List[Tuple[int, int, int, int]] = []
    for dst, head in enumerate(_rank_heads(h, reader_tp, reader_rank)):
        if writer_tp >= h:
            w, src = head * writer_tp // h, 0  # the first rank holding it
        else:
            per = h // writer_tp
            w, src = head // per, head % per
        last = out[-1] if out else None
        if last and last[0] == w and last[1] + last[3] == src and last[2] + last[3] == dst:
            out[-1] = (w, last[1], last[2], last[3] + 1)
        else:
            out.append((w, src, dst, 1))
    assert len({s[3] for s in out}) == 1
    return out


def page_key(model: str, layer, kind: str, tp_rank: int, page_hash: str) -> str:
    """Key of one page: model / layer (or ``ALL_LAYERS``) / K|V|KV / TP rank / chained
    prefix hash."""
    return f"{model}/L{layer}/{kind}/tp{tp_rank}/{page_hash}"
