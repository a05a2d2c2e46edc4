"""Inputs and the reference computation shared by the tests of the numpy-fallback types (csrc/fallback.cuh).

The reference is the reference package's `else` branch (dequant.py:24-28): `gguf.quants.dequantize(bytes, qtype)` in numpy,
then `torch.from_numpy(...).to(dtype)`."""
import numpy as np
import torch
import gguf

Q = gguf.GGMLQuantizationType
FALLBACK = [Q.IQ2_XXS, Q.IQ2_XS, Q.IQ2_S, Q.IQ3_XXS, Q.IQ3_S, Q.IQ1_S, Q.IQ1_M, Q.TQ1_0, Q.TQ2_0, Q.MXFP4, Q.NVFP4]
TORCH_DT = {0: torch.float16, 1: torch.bfloat16, 2: torch.float32}

# byte offset of the block's f16 scale (IQ1_M spreads it over four nibbles; the FP4 types have 8-bit scales)
_F16_SCALE_AT = {Q.IQ2_XXS: 0, Q.IQ2_XS: 0, Q.IQ2_S: 0, Q.IQ3_XXS: 0, Q.IQ3_S: 0, Q.IQ1_S: 0, Q.TQ1_0: 52, Q.TQ2_0: 64}
# f16 scales that exercise the edges of the arithmetic: +-Inf, NaN, zeros, subnormals, the largest finite value
F16_SPECIALS = [0x7C00, 0xFC00, 0x7E00, 0xFE01, 0x0000, 0x8000, 0x0001, 0x03FF, 0x8200, 0x7BFF, 0x3C00]
MXFP4_SPECIALS = [0, 1, 2, 126, 127, 128, 254, 255]
NVFP4_SPECIALS = [0x00, 0x7F, 0xFF, 0x01, 0x07, 0x08, 0x80, 0x81, 0x87, 0xF8, 0x7E, 0x38]


def _set_f16_scale(blocks, qt, bits):
    """Write the f16 scale field of every row of `blocks` ([n, type_size] uint8) to the patterns `bits` ([n])."""
    bits = np.asarray(bits, dtype=np.uint16)
    if qt == Q.IQ1_M:
        words = blocks[:, 48:56].copy().view(np.uint16)                      # [n, 4]
        for k in range(4):
            words[:, k] = (words[:, k] & 0x0FFF) | (((bits >> (4 * k)) & 0xF) << 12)
        blocks[:, 48:56] = words.view(np.uint8)
    else:
        at = _F16_SCALE_AT[qt]
        blocks[:, at:at + 2] = bits.reshape(-1, 1).view(np.uint8).reshape(-1, 2)


def random_blocks(qt, n_blocks, seed=0, scale=None, specials=False):
    """[n_blocks, type_size] uint8.  Raw random bytes; with `scale` every block scale is a finite value of about that size
    (so Linear outputs stay finite); with `specials` the first blocks carry the edge-case scales above."""
    _bs, ts = gguf.GGML_QUANT_SIZES[qt]
    rng = np.random.default_rng(seed + 1000 * int(qt))
    blocks = rng.integers(0, 256, size=(n_blocks, ts), dtype=np.uint8)
    if scale is not None:
        if qt == Q.MXFP4:        # d = 2^(e - 128): e near 128 + log2(scale)
            e0 = int(np.clip(np.round(np.log2(scale)) + 128, 2, 250))
            blocks[:, 0] = rng.integers(e0 - 1, e0 + 2, size=n_blocks)
        elif qt == Q.NVFP4:      # ue4m3 / 2 = (8 + m) 2^(e - 11): exponent field near 11 + log2(scale / 8)
            e = int(np.clip(np.round(np.log2(scale / 8.0)) + 11, 1, 14))
            blocks[:, 0:4] = (e << 3) | rng.integers(0, 8, size=(n_blocks, 4))
        else:
            mags = (rng.uniform(0.5, 1.5, size=n_blocks) * scale).astype(np.float16)
            _set_f16_scale(blocks, qt, mags.view(np.uint16))
    if specials:
        if qt == Q.MXFP4:
            k = min(n_blocks, len(MXFP4_SPECIALS))
            blocks[:k, 0] = MXFP4_SPECIALS[:k]
        elif qt == Q.NVFP4:
            k = min(n_blocks, len(NVFP4_SPECIALS))
            for j in range(4):
                blocks[:k, j] = np.roll(NVFP4_SPECIALS, j)[:k]
        else:
            k = min(n_blocks, len(F16_SPECIALS))
            _set_f16_scale(blocks[:k], qt, F16_SPECIALS[:k])        # a view: writes through
    return blocks


def gguf_values(blocks, qt):
    """gguf-py's fp32 values of the packed bytes, flat."""
    return gguf.quants.dequantize(np.ascontiguousarray(blocks).reshape(-1), qt).reshape(-1)


def reference_tensor(blocks, qt, out_code):
    """The reference's result: torch.from_numpy(gguf.quants.dequantize(...)).to(dtype), flat, on the CPU."""
    return torch.from_numpy(gguf_values(blocks, qt)).to(TORCH_DT[out_code])
