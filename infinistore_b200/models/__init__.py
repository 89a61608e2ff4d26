"""KV-cache shapes of the model families the store is deployed with, and a paged KV cache
whose pages map 1:1 onto store blocks.

The reference is model-agnostic (it moves opaque byte blocks; its only "model" is the toy
nn.Sequential of example/demo_prefill.py:21-48).  What callers need from a KV store is the
page geometry (bytes per page per layer), a key scheme that encodes layer / TP rank /
prefix hash (docs/source/design.rst:50) and layer-wise streaming; this package provides
those for real model configurations - plus the two consumer-side shapes the device read
kernels serve directly: a head-major decode cache filled by the layout-swizzling read
(``HeadMajorKVCache``) and several caches of one GPU filled by one fetch (``read_layer_multi``).
"""
from .kv_layout import (KVLayout, LAYOUTS, MLA_LAYOUTS, MLALayout, get_layout, chain_hashes,
                        mla_chunk_key, mla_page_key, mla_segment_key, page_key, segment_key)
from .paged_kv import HeadMajorKVCache, MLAKVCache, PagedKVCache, layer_keys, read_layer_multi

__all__ = ["KVLayout", "LAYOUTS", "get_layout", "chain_hashes", "page_key", "PagedKVCache",
           "HeadMajorKVCache", "layer_keys", "read_layer_multi", "MLALayout", "MLA_LAYOUTS",
           "mla_page_key", "mla_chunk_key", "MLAKVCache", "segment_key", "mla_segment_key"]
