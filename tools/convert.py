"""Convert a diffusion-model checkpoint (.safetensors / .ckpt / .pt / .pth / .bin) to GGUF, optionally quantised on the GPU, or
quantise a GGUF file.

    python tools/convert.py --src flux1-dev.safetensors                      # F16 / BF16 file, as the reference's convert.py
    python tools/convert.py --src flux1-dev.safetensors --qtype Q8_0         # quantised in the same run (needs a CUDA device)

    python tools/convert.py --src flux1-dev.safetensors --qtype Q4_K_S       # a llama-quantize K mixture, also on the GPU

    python tools/convert.py --src flux1-dev-BF16.gguf --qtype Q4_K_S         # a GGUF input: llama-quantize's step, on the GPU
    python tools/convert.py --src flux1-dev-Q8_0.gguf --qtype Q4_K_S --allow-requantize
    python tools/convert.py --src wan2.1-BF16.gguf --qtype Q4_K_S --fix-5d fix_5d_tensors_wan.safetensors

A .gguf --src needs --qtype.  Its tensors keep their type and bytes wherever the rules leave them alone; an already quantised
tensor the rules would change is refused unless --allow-requantize, which decodes it on the GPU and quantises it again.  A wan /
hyvid file from the reference's convert.py lacks its 5-D weight: --fix-5d merges the fix_5d_tensors_<arch>.safetensors that
convert.py left beside it.

--qtype: F16, BF16, Q8_0, Q5_1, Q5_0, Q4_1 or Q4_0, or one of llama-quantize's K mixtures Q2_K, Q3_K_S, Q3_K_M, Q3_K_L, Q4_K_S,
Q4_K_M, Q5_K_S, Q5_K_M or Q6_K.  See comfyui-gguf_b200/convert.py for the type policy.
"""
import argparse
import logging
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main(argv=None):
    import __graft_entry__ as ge
    convert = ge._sub("convert")
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--src", required=True, help="source checkpoint")
    ap.add_argument("--dst", help="output .gguf (default: <src>-<type>.gguf; '{ftype}' is replaced by the type name)")
    ap.add_argument("--qtype", choices=sorted(convert.QTYPES) + sorted(convert.KQUANT_MIXTURES), help="quantise to this type (default: the F16 / BF16 file)")
    ap.add_argument("--overwrite", action="store_true", help="replace an existing output file")
    ap.add_argument("--allow-requantize", action="store_true", help="GGUF input: quantise already quantised tensors again")
    ap.add_argument("--fix-5d", metavar="PATH", help="GGUF input: merge this fix_5d_tensors_<arch>.safetensors side file")
    args = ap.parse_args(argv)
    if not os.path.isfile(args.src):
        ap.error(f"no such file: {args.src}")
    is_gguf = args.src.lower().endswith(".gguf")
    if is_gguf and args.qtype is None:
        ap.error("a .gguf --src needs --qtype")
    if not is_gguf and (args.allow_requantize or args.fix_5d):
        ap.error("--allow-requantize and --fix-5d apply to a .gguf --src only")
    logging.basicConfig(level=logging.INFO, format="%(message)s")
    if is_gguf:
        res = convert.convert_gguf_file(args.src, args.dst, args.qtype, overwrite=args.overwrite,
                                        allow_requantize=args.allow_requantize, fix_5d=args.fix_5d)
    else:
        res = convert.convert_file(args.src, args.dst, args.qtype, overwrite=args.overwrite)
    counts = {}
    for p in res.plans:
        counts[p.qtype.name] = counts.get(p.qtype.name, 0) + 1
    print(f"wrote {res.path} [arch {res.arch.name}]: " + ", ".join(f"{k} ({v})" for k, v in counts.items())
          + " | " + ", ".join(f"{k} {v:.2f} s" for k, v in res.seconds.items()))


if __name__ == "__main__":
    main()
