#!/usr/bin/env python
"""Generate the golden vectors of the numpy-fallback types from the installed gguf-py.

    python tests/golden/make_golden_fallback.py

For each of the eleven types the reference dequantises through `gguf.quants.dequantize` (reference dequant.py:24-28), writes

    fallback_<QTYPE>.npz    blocks: [n, type_size] uint8 (seeded random bytes, edge-case scales in the first rows)
                            f32:    gguf-py's fp32 values, flat

These pin gguf-py's own output: tests/test_fallback_types.py checks that the installed gguf-py still produces `f32` (a gguf
upgrade that changes the arithmetic is noticed), and tests/test_gpu_fallback_types.py checks the GPU kernel against them.
"""
import os
import sys

import gguf
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from fallback_cases import FALLBACK, gguf_values, random_blocks  # noqa: E402

N_BLOCKS = {32: 48, 64: 32}     # by block size; 256-element types: 12 blocks


def main():
    for qt in FALLBACK:
        bs, _ts = gguf.GGML_QUANT_SIZES[qt]
        blocks = random_blocks(qt, N_BLOCKS.get(bs, 12), seed=20261016, specials=True)
        path = os.path.join(HERE, f"fallback_{qt.name}.npz")
        np.savez_compressed(path, blocks=blocks, f32=gguf_values(blocks, qt))
        print("wrote", path)


if __name__ == "__main__":
    main()
