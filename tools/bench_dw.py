"""Micro-benchmark of the HBM/issue-bound kernels of a ConvNeXt block front half on the ConvNeXt-L@800x1280 shapes: uc_dwconv7
(fp32-FMA TMA kernel) with and without LayerNorm statistics, uc_dwconv7_mma (tensor cores) and uc_layernorm — timed as
back-to-back CUDA-graph kernel nodes (CUDA events around a replay), working set L2 resident like in the frame."""
import os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from unicorn_b200 import ops
dev = "cuda"
SHAPES = [("s1", 200, 320, 192), ("s2", 100, 160, 384), ("s3", 50, 80, 768), ("s4", 25, 40, 1536), ("head0", 100, 160, 256),
          ("head1", 50, 80, 256), ("head2", 25, 40, 256), ("mot.s3", 96, 128, 768)]
R = 20
HBM = float(os.environ.get("UC_HBM_GBS", 6487.1))


CTR = torch.zeros(R + 1, dtype=torch.int32, device=dev)  # one zeroed work counter per launch of a replay


def timed(fn):
    CTR.zero_(); fn(R); torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        CTR.zero_()
        for k in range(R): fn(k)
    g.replay(); torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); g.replay(); g.replay(); b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) * 1e3 / (2 * R)


ONLY = [a for a in sys.argv[1:]]
for name, H, W, C in SHAPES:
    if ONLY and name not in ONLY:
        continue
    x = torch.randn(1, H, W, C, device=dev).bfloat16()
    w = ops.pack_dw_weight(torch.randn(C, 1, 7, 7, device=dev) / 7)
    b, lw, lb = (torch.randn(C, device=dev) for _ in range(3))
    y = torch.empty_like(x)
    st = torch.zeros(H * W, 2, dtype=torch.int64, device=dev)
    t_dw = timed(lambda k: ops.dwconv7(x, w, b, out=y, work_counter=CTR[k:k + 1]))
    t_static = timed(lambda k: ops.dwconv7(x, w, b, out=y))
    t_st = timed(lambda k: ops.dwconv7(x, w, b, out=y, ln_stats=st, work_counter=CTR[k:k + 1]))
    wf = ops.pack_dw_weight_mma(torch.randn(C, 1, 7, 7, device=dev) / 7, b)
    t_mma = timed(lambda k: ops.dwconv7_mma(x, wf, out=y, work_counter=CTR[k:k + 1]))
    t_ln = timed(lambda k: ops.layernorm(y.view(-1, C), lw, lb, 1e-6, out=y.view(-1, C)))
    byt = 4.0 * H * W * C  # algorithmic bytes: read + write the bf16 map once
    fl = 98.0 * H * W * C
    print(f"{name:7s} {H:4d}x{W:<4d} C={C:5d}  dwconv {t_dw:7.1f} us ({byt/t_dw/1e3:7.1f} GB/s = {byt/t_dw/1e3/HBM*100:5.1f}% HBM, {fl/t_dw/1e6:5.1f} TFLOP/s fp32)"
          f"  MMA {t_mma:7.1f} us ({byt/t_mma/1e3/HBM*100:5.1f}% HBM)  static-schedule {t_static:7.1f} us  +stats {t_st:7.1f} us  layernorm {t_ln:6.1f} us", flush=True)
