#!/usr/bin/env python
"""Generate the reference stage-1 GGUF fixtures from the UNMODIFIED reference converter.

Run in the build container only (needs /root/reference, which does not exist on
the GPU box):   python tests/golden/make_golden_stage1.py

What is produced (all under tests/golden/):
  stage1_flux.gguf, stage1_sdxl.gguf, stage1_wan.gguf   the reference's tools/convert.py
                        run on the seeded checkpoints of tests/convert_gguf_cases.py
                        (flux bf16, sdxl fp16 with `comfy.gguf.orig_shape` fields, wan bf16)
  fix_5d_tensors_wan.safetensors   the side file the reference writes for wan's
                        5-D patch embedding, which its stage-1 file leaves out

The reference script is run by path, unchanged, in a temporary working directory:
it writes the side file into the current directory and refuses to overwrite one.
"""
import os
import shutil
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
REF_CONVERT = "/root/reference/tools/convert.py"

import convert_gguf_cases as cc  # noqa: E402


def main():
    from safetensors.torch import save_file
    for arch, dt in cc.FIXTURES.items():
        with tempfile.TemporaryDirectory(prefix="stage1_") as tmp:
            src = os.path.join(tmp, f"{arch}.safetensors")
            save_file(cc.checkpoint(arch, dt), src)
            dst = os.path.join(tmp, f"{arch}.gguf")
            subprocess.run([sys.executable, REF_CONVERT, "--src", src, "--dst", dst], cwd=tmp, check=True)
            shutil.copyfile(dst, cc.fixture_path(arch))
            fix = os.path.join(tmp, f"fix_5d_tensors_{arch}.safetensors")
            if os.path.isfile(fix):
                shutil.copyfile(fix, os.path.join(HERE, os.path.basename(fix)))
            print(f"wrote {cc.fixture_path(arch)}" + (f" and {os.path.basename(fix)}" if os.path.isfile(fix) else ""))


if __name__ == "__main__":
    main()
