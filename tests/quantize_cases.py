"""Inputs shared by the quantiser tests (tests/test_quantize.py, tests/test_gpu_quantize.py): seeded blocks and the blocks
where gguf-py's quantisers are easiest to get wrong, plus synthetic key sets of the eleven converter architectures."""
import gguf
import numpy as np

Q = gguf.GGMLQuantizationType
QUANT_TYPES = [Q.Q4_0, Q.Q4_1, Q.Q5_0, Q.Q5_1, Q.Q8_0, Q.BF16]


def seeded_blocks(n, seed):
    """n blocks of 32 fp32 values at scales from 1e-3 to 1e2, with an occasional outlier."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, 32)).astype(np.float32) * np.float32(10.0) ** rng.integers(-3, 3, size=(n, 1)).astype(np.float32)
    out = rng.random((n, 32)) < 0.01
    x[out] *= np.float32(20.0)
    return x.astype(np.float32)


def adversarial_blocks():
    """[n, 32] fp32, every row finite."""
    rows = []
    r = np.random.default_rng(11)
    base = (r.standard_normal(32) * 0.1).astype(np.float32)
    for i, j in ((0, 5), (3, 31), (30, 31)):
        for si, sj in ((1, -1), (-1, 1), (1, 1), (-1, -1)):
            b = base.copy()
            b[i], b[j] = si * 0.75, sj * 0.75           # a tie for the largest |x| with mixed signs
            rows.append(b)
    for v in (1.0, -1.0, 3.3, -7e-3, 65504.0, 1e-6):
        rows.append(np.full(32, v, np.float32))          # all equal
    rows.append(np.zeros(32, np.float32))
    rows.append(np.full(32, -0.0, np.float32))
    for k in range(6):                                   # zeros of both signs, alone or next to one-signed values
        z = np.where(r.random(32) < 0.5, np.float32(0.0), np.float32(-0.0)).astype(np.float32)
        if k >= 2:
            m = r.random(32) < 0.3
            z[m] = (np.abs(r.standard_normal(m.sum())) + 0.1) * (1 if k % 2 else -1)
        rows.append(z)
    for pos in (0, 7, 16, 31):                           # a single nonzero element
        for v in (2.5, -2.5, 1e-30):
            b = np.zeros(32, np.float32)
            b[pos] = v
            rows.append(b)
    for s in (1.0, -1.0):                                # codes 16 / 32 before the clip: +max and -max in one block
        b = (base * 0.5).astype(np.float32)
        b[4], b[20] = s * 1.0, -s * 1.0
        rows.append(b)
    b = np.linspace(-1, 1, 32, dtype=np.float32)
    rows.append(b)
    rows.append(-b)
    for scale in (1e-38, 1e-39, 1e-41, 1e-44, 1.4e-45, 2.0 ** -126, 2.0 ** -129):   # subnormal values and scales
        rows.append((r.standard_normal(32) * scale).astype(np.float32))
        rows.append(np.full(32, scale, np.float32))
    t = np.zeros(32, np.float32)
    t[3] = np.float32(2.0 ** -126)
    rows.append(t)
    for scale in (1e5, 1e6, 3e38):                      # scales that overflow fp16 (and max - min that overflows fp32)
        rows.append((r.standard_normal(32) * scale).clip(-3.3e38, 3.3e38).astype(np.float32))
    b = np.zeros(32, np.float32)
    b[0], b[1] = 3.0e38, -3.0e38
    rows.append(b)
    rows.append(np.full(32, 3.4e38, np.float32))
    for k in range(8):                                   # values on the rounding edges of x / d + 0.5
        b = (np.arange(32) - 16).astype(np.float32) * np.float32(0.5 + k * 0.25)
        rows.append(b)
    return np.stack(rows).astype(np.float32)


def gguf_bytes(x, qtype):
    """gguf-py's bytes for fp32 values x [..., K]."""
    return gguf.quants.quantize(np.ascontiguousarray(x, dtype=np.float32), qtype)


# ---------------------------------------------------------------- synthetic key sets for the converter's architecture table
ARCH_KEYS = {
    "flux": ["double_blocks.0.img_attn.proj.weight", "img_in.weight"],
    "sd3": ["joint_blocks.0.x_block.attn.qkv.weight", "pos_embed"],
    "aura": ["double_layers.3.modX.1.weight", "init_x_linear.weight"],
    "hidream": ["caption_projection.0.linear.weight", "double_stream_blocks.0.block.ff_i.shared_experts.w3.weight"],
    "cosmos": ["blocks.0.mlp.layer1.weight", "blocks.0.adaln_modulation_cross_attn.1.weight"],
    "ltxv": ["adaln_single.emb.timestep_embedder.linear_2.weight", "transformer_blocks.27.scale_shift_table",
             "caption_projection.linear_2.weight"],
    "hyvid": ["double_blocks.0.img_attn_proj.weight", "txt_in.individual_token_refiner.blocks.1.self_attn_qkv.weight"],
    "wan": ["blocks.0.self_attn.norm_q.weight", "text_embedding.2.weight", "head.modulation"],
    "sdxl": ["input_blocks.3.0.op.weight", "input_blocks.6.0.op.weight", "output_blocks.2.2.conv.weight",
             "output_blocks.5.2.conv.weight", "label_emb.0.0.weight"],
    "sd1": ["input_blocks.3.0.op.weight", "input_blocks.6.0.op.weight", "input_blocks.9.0.op.weight",
            "output_blocks.2.1.conv.weight", "output_blocks.5.2.conv.weight", "output_blocks.8.2.conv.weight"],
    "lumina2": ["cap_embedder.1.weight", "context_refiner.0.attention.qkv.weight"],
}
