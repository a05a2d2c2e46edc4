"""Compare two GGUF files tensor by tensor: type, shape and whether the bytes are equal.

    python tools/compare_gguf.py ours.gguf theirs.gguf

Useful to check a file this package converted against one written by llama-quantize (for example the K mixtures against a
b3962 build with the image-model patch), or any two conversions of the same checkpoint.  Prints one line per tensor name found
in either file and a summary; the exit code is 0 when both files hold the same tensors with equal types, shapes and bytes.
"""
import argparse
import sys

import gguf
import numpy as np


def tensors(path):
    r = gguf.GGUFReader(path)
    return {t.name: (gguf.GGMLQuantizationType(t.tensor_type).name, tuple(int(d) for d in t.shape),
                     np.asarray(t.data).view(np.uint8).reshape(-1)) for t in r.tensors}


def compare(a_path, b_path, out=sys.stdout):
    a, b = tensors(a_path), tensors(b_path)
    names = list(a) + [n for n in b if n not in a]
    width = max((len(n) for n in names), default=4)
    same = 0
    for n in names:
        ta, tb = a.get(n), b.get(n)
        if ta is None or tb is None:
            print(f"{n:<{width}}  only in {'B' if ta is None else 'A'}", file=out)
            continue
        types = ta[0] if ta[0] == tb[0] else f"{ta[0]} / {tb[0]}"
        shapes = "x".join(map(str, ta[1])) if ta[1] == tb[1] else f"{'x'.join(map(str, ta[1]))} / {'x'.join(map(str, tb[1]))}"
        equal = ta[0] == tb[0] and ta[1] == tb[1] and np.array_equal(ta[2], tb[2])
        if not equal and ta[2].size == tb[2].size:
            detail = f"differ ({int(np.count_nonzero(ta[2] != tb[2]))} of {ta[2].size} bytes)"
        else:
            detail = "equal" if equal else "differ"
        same += equal
        print(f"{n:<{width}}  {types:<12} {shapes:<20} {detail}", file=out)
    print(f"{same} of {len(names)} tensors equal", file=out)
    return same == len(names)


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("a")
    ap.add_argument("b")
    args = ap.parse_args(argv)
    return 0 if compare(args.a, args.b) else 1


if __name__ == "__main__":
    sys.exit(main())
