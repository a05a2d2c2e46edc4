"""Backward of the packed-weight Linear (dX = dY . W) at the Flux shapes, and the peak memory of a training step through a
Flux-shape block stack.

Per (N, K) and M, CUDA-graph replays over rotated weight copies (as tools/bench_linear.py --graph), in milliseconds:
  grad_input   ggufb200_linear_grad_input: K1 dequant into a workspace + the MN-major dense GEMM (what the layer's backward runs)
  k1           the K1 dequant alone (its share of grad_input)
  k1_matmul    K1 + torch.matmul(dY, W) (cuBLAS on the dequantised weight)
  ref_bwd      the reference's backward: F.linear autograd on the weight of oracle/torch_chain.py's dequant chain, saved from the
               forward (timed with events, not in a graph: torch.autograd.grad of the recorded forward)
Then the peak allocated memory of forward + backward through 4 Flux double-block-shaped stacks of GGMLOps.Linear layers with the
input requiring grad: the packed route (nothing dense saved) and the two-step route (F.linear saves every dequantised W).
Prints the card's name and power limit first: the numbers belong to them."""
import argparse
import os
import subprocess
import sys

import gguf
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as ge  # noqa: E402
import oracle  # noqa: E402
from oracle import torch_chain  # noqa: E402

SHAPES = [(3072, 3072), (9216, 3072), (12288, 3072), (3072, 12288)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        return f"{name}, {q.stdout.strip()}"
    except (OSError, subprocess.SubprocessError):
        return f"{name}, power limit unknown"


def graph_ms(fn, iters=10, per=8):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(per):
            fn()
    g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / (iters * per)


def event_ms(fn, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def packed_copies(ops, qt, N, K, copies, dev):
    bs, ts = gguf.GGML_QUANT_SIZES[qt]
    out = []
    for c in range(copies):
        chunk = min(N * K // bs, 1 << 15)
        raw = torch.from_numpy(oracle.random_blocks(int(qt), chunk, seed=c, scale=0.02))
        packed = raw.repeat((N * K // bs + chunk - 1) // chunk, 1)[: N * K // bs].reshape(N, K // bs * ts).contiguous().to(dev)
        out.append(ops.GGMLTensor(packed, tensor_type=qt, tensor_shape=torch.Size((N, K))))
    return out


def times(ops, dq, qt, act, M, N, K, copies, dev):
    ws = packed_copies(ops, qt, N, K, copies, dev)
    raws = [w.as_subclass(torch.Tensor) for w in ws]
    dy = torch.randn(M, N, device=dev, dtype=act)
    state = {"i": 0}

    def nxt():
        state["i"] = (state["i"] + 1) % len(ws)
        return state["i"]
    math = 0
    row = {
        "grad_input": graph_ms(lambda: ops.linear_grad_input(dy, raws[nxt()], qt, N, K, math)),
        "k1": graph_ms(lambda: dq.dequantize_tensor(ws[nxt()], act)),
        "k1_matmul": graph_ms(lambda: torch.matmul(dy, dq.dequantize_tensor(ws[nxt()], act))),
    }
    x = torch.randn(M, K, device=dev, dtype=act, requires_grad=True)
    W = torch_chain.dequantize_tensor(raws[0], int(qt), (N, K), act)
    y = torch.nn.functional.linear(x, W)
    row["ref_bwd"] = event_ms(lambda: torch.autograd.grad(y, x, dy, retain_graph=True))
    got = ops.linear_grad_input(dy, raws[0], qt, N, K, math)
    want = dy.double() @ dq.dequantize_tensor(ws[0], act).double()
    row["rel_err"] = float((got.double() - want).norm() / want.norm())
    return row


def stack_peak(ops, qt, act, M, dev, two_step):
    D = 3072
    blocks = []
    for b in range(4):
        blocks.append([])
        for N, K in ((9216, D), (D, D), (12288, D), (D, 12288)):
            lin = ops.GGMLOps.Linear(K, N)
            lin.load_state_dict({"weight": packed_copies(ops, qt, N, K, 1, dev)[0]})
            blocks[-1].append(lin)
    saved = ops.GGMLOps.Linear._fused_ok
    if two_step:
        ops.GGMLOps.Linear._fused_ok = lambda self, x: False
    try:
        x = torch.randn(M, D, device=dev, dtype=act, requires_grad=True)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        h = x
        for qkv, proj, mlp0, mlp2 in blocks:
            h = h + proj(qkv(h)[:, :D])
            h = h + mlp2(torch.nn.functional.gelu(mlp0(h)))
        h.float().square().mean().backward()
        torch.cuda.synchronize()
        return (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    finally:
        ops.GGMLOps.Linear._fused_ok = saved


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--qtype", default="Q4_K")
    ap.add_argument("--M", type=int, nargs="+", default=[512, 4096])
    ap.add_argument("--copies", type=int, default=4)
    args = ap.parse_args()
    ops, dq = ge._sub("ops"), ge._sub("dequant")
    dev = torch.device("cuda:0")
    qt = gguf.GGMLQuantizationType[args.qtype]
    act = torch.bfloat16
    print(f"card: {card()}")
    print(f"{args.qtype} bf16, ms per call (CUDA-graph replays; ref_bwd with events)")
    print(f"{'N':>6} {'K':>6} {'M':>5} {'grad_input':>10} {'k1':>8} {'k1_share':>8} {'k1_matmul':>9} {'ref_bwd':>8} {'rel_err':>9}")
    for N, K in SHAPES:
        for M in args.M:
            r = times(ops, dq, qt, act, M, N, K, args.copies, dev)
            print(f"{N:>6} {K:>6} {M:>5} {r['grad_input']:>10.4f} {r['k1']:>8.4f} {r['k1'] / r['grad_input']:>8.2f} {r['k1_matmul']:>9.4f} "
                  f"{r['ref_bwd']:>8.4f} {r['rel_err']:>9.2e}")
    for M in args.M:
        packed = stack_peak(ops, qt, act, M, dev, False)
        two = stack_peak(ops, qt, act, M, dev, True)
        print(f"peak memory, forward + backward, 4 Flux-shape blocks (16 Linears), M = {M}: packed {packed:.2f} GiB, two-step {two:.2f} GiB")


if __name__ == "__main__":
    main()
