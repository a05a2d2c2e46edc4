"""Seeded tiny checkpoints shared by the GGUF-input converter tests (tests/test_convert_gguf.py, tests/test_gpu_convert_gguf.py)
and by tests/golden/make_golden_stage1.py, which runs the reference's stage 1 on three of them.

Each checkpoint mixes the tensor kinds the type rules tell apart: the main dtype (bf16 or fp16, which makes the stage-1 file
BF16 or F16), fp32 matrices (stage 1 F16) and small or 1-D fp32 tensors (F32), keep-listed names, rows that are not a multiple
of 256 (the K mixtures' F16 fallback) or of 32 (never quantised), attention-value / fused-qkv / ffn_down names, the SD1 / SDXL
reshape with its `comfy.gguf.orig_shape` field, and wan's 5-D patch embedding."""
import os

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden")
ARCHES = ("flux", "sd3", "sdxl", "wan")
# the reference stage-1 fixtures: (architecture, main dtype) -> tests/golden/stage1_<arch>.gguf
FIXTURES = {"flux": torch.bfloat16, "sdxl": torch.float16, "wan": torch.bfloat16}
FIX_5D = os.path.join(GOLDEN, "fix_5d_tensors_wan.safetensors")


def fixture_path(arch):
    return os.path.join(GOLDEN, f"stage1_{arch}.gguf")


def checkpoint(arch: str, dt: torch.dtype) -> dict:
    """The seeded checkpoint of `arch` whose matrices are `dt` (bf16 or fp16), in a fixed key order."""
    g = torch.Generator().manual_seed(1000 + ARCHES.index(arch) * 10 + (dt == torch.float16))
    f32 = lambda *s: torch.randn(*s, generator=g) * 0.02
    r = lambda *s: f32(*s).to(dt)
    if arch == "flux":
        return {
            "img_in.weight": r(64, 64),
            "img_in.bias": r(64),
            "double_blocks.0.img_attn.qkv.weight": r(96, 256),
            "double_blocks.0.img_attn.proj.weight": r(64, 256),
            "double_blocks.0.img_attn.proj.bias": r(64),
            "double_blocks.0.img_attn.norm.key_norm.scale": f32(128),
            "double_blocks.0.img_mlp.0.weight": r(128, 256),
            "double_blocks.0.img_mlp.2.weight": r(64, 512),
            "single_blocks.0.linear2.weight": f32(64, 512),
            "double_blocks.0.odd.weight": r(64, 96),
            "double_blocks.0.odd2.weight": r(32, 48),
            "double_blocks.0.small.weight": f32(16, 16),
            "final_layer.linear.weight": r(64, 256),
        }
    if arch == "sd3":
        return {
            "x_embedder.proj.weight": r(64, 16, 2, 2),
            "pos_embed": r(1, 64, 256),
            "joint_blocks.0.x_block.attn.qkv.weight": r(96, 256),
            "joint_blocks.0.x_block.attn.proj.weight": r(64, 256),
            "joint_blocks.0.x_block.mlp.fc2.weight": r(64, 512),
            "joint_blocks.0.context_block.attn.qkv.weight": r(96, 256),
            "joint_blocks.0.context_block.attn.qkv.bias": f32(96),
            "joint_blocks.0.x_block.odd.weight": r(64, 160),
            "proj_out.weight": r(64, 256),
        }
    if arch == "sdxl":
        sd = {k: r(64, 4, 1, 1) for k in ("input_blocks.3.0.op.weight", "input_blocks.6.0.op.weight",
                                         "output_blocks.2.2.conv.weight", "output_blocks.5.2.conv.weight", "label_emb.0.0.weight")}
        sd.update({
            "input_blocks.0.0.weight": r(32, 4, 3, 3),
            "input_blocks.1.0.in_layers.2.weight": r(32, 32, 3, 3),                          # reshaped to [36, 256]
            "input_blocks.4.1.proj_in.weight": r(80, 320),                                   # reshaped to [100, 256]
            "input_blocks.4.1.transformer_blocks.0.attn1.to_v.weight": r(64, 256),
            "input_blocks.4.1.transformer_blocks.0.attn2.to_v.weight": r(64, 512),
            "input_blocks.4.1.transformer_blocks.0.attn1.to_q.weight": r(64, 256),
            "input_blocks.4.1.transformer_blocks.0.ff.net.2.weight": r(64, 512),
            "input_blocks.4.1.norm.weight": r(64, 40),                                       # rows of 40, not reshaped
            "time_embed.0.weight": f32(256, 64),
            "time_embed.0.bias": f32(256),
        })
        return sd
    if arch == "wan":
        return {
            "patch_embedding.weight": r(64, 16, 1, 2, 2),
            "patch_embedding.bias": r(64),
            "text_embedding.2.weight": r(64, 256),
            "blocks.0.modulation": f32(1, 6, 256),
            "blocks.0.self_attn.q.weight": r(64, 256),
            "blocks.0.self_attn.v.weight": r(64, 256),
            "blocks.0.self_attn.v.bias": r(64),
            "blocks.0.self_attn.norm_q.weight": r(256),
            "blocks.0.cross_attn.v.weight": r(64, 256),
            "blocks.0.ffn.0.weight": r(128, 256),
            "blocks.0.ffn.2.weight": r(64, 512),
            "blocks.1.self_attn.v.weight": r(64, 256),
            "blocks.1.cross_attn.v.weight": r(64, 96),
            "head.modulation": f32(1, 2, 256),
            "head.head.weight": r(64, 256),
        }
    raise KeyError(arch)
