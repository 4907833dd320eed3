"""NV12 input path on one GPU, seeded weights.

    python tools/bench_nv12.py [--launches 2000] [--steps 30] [--warmup 5] [--rounds 5]

Kernel lines: uc_letterbox_nv12 against uc_letterbox_u8 (RGB in, BGR out) for 1080x1920 and 480x640 frames letterboxed into 800x1280,
`launches` launches captured in one CUDA graph and timed with CUDA events; the two kernels alternate over `rounds` rounds and the
median per launch is reported.  SOT lines: UnicornSOTBatch(unicorn_track_large, 800x1280, device_preproc=True).track on 1080x1920
frames in pinned host memory, NV12 against RGB, at n_seq = 1 and 4; a step is synchronous (upload, letterbox, graph replay,
read-back), timed with a host clock over `steps` steps; the two formats alternate over `rounds` rounds on the same driver, and the
best round is reported as frames/s with the bytes one step copies to the device.  Host line: cv2.cvtColor(COLOR_YUV2RGB_NV12) plus
sot.preprocess of one 1080x1920 frame on the host CPU, the work an NV12 caller no longer does.  The card name and power limit are read
in the same run.  One JSON line per result."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def graph_of(fn, reps):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    torch.cuda.synchronize()
    return g


def time_graph(g):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    g.replay()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def kernels(args, card):
    from unicorn_b200 import ops, shared_ops
    H, W = 800, 1280
    out = torch.empty(1, H, W, 3, dtype=torch.uint8, device="cuda")
    for h, w in [(1080, 1920), (480, 640)]:
        nv12 = torch.randint(0, 256, (h * 3 // 2, w), dtype=torch.uint8, device="cuda")
        rgb = torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, device="cuda")
        graphs = {"uc_letterbox_nv12": graph_of(lambda: shared_ops.letterbox_nv12(nv12, (H, W), out=out), args.launches),
                  "uc_letterbox_u8": graph_of(lambda: ops.letterbox_u8(rgb, (H, W), swap_rb=True, out=out), args.launches)}
        us = {k: [] for k in graphs}
        for _ in range(args.rounds):
            for k, g in graphs.items():
                us[k].append(time_graph(g) * 1e3 / args.launches)
        for k, v in us.items():
            print(json.dumps({"bench": "kernel", "kernel": k, "src": f"{h}x{w}", "dst": f"{H}x{W}", "us_per_launch": round(statistics.median(v), 2),
                              "rounds_us": [round(x, 2) for x in v], "launches": args.launches, "card": card}), flush=True)


def sot(args, card):
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.sot import UnicornSOTBatch
    from unicorn_b200.weights import make_state_dict
    name, (H, W), (h, w) = "unicorn_track_large", (800, 1280), (1080, 1920)
    eng = UnicornEngine(make_state_dict(name, 0), name)
    g = torch.Generator().manual_seed(0)
    rgb = torch.randint(0, 256, (h, w, 3), dtype=torch.uint8, generator=g).pin_memory()
    nv12 = torch.randint(0, 256, (h * 3 // 2, w), dtype=torch.uint8, generator=g).pin_memory()
    for n in (1, 4):
        b = UnicornSOTBatch(eng, (H, W), n, device_preproc=True)
        for i in range(n):
            b.initialize(i, rgb, {"init_bbox": [700, 400, 300, 200]})
        fps = {"rgb": [], "nv12": []}
        frames = {"rgb": [rgb] * n, "nv12": [nv12] * n}
        for k in fps:
            for _ in range(args.warmup):
                b.track(frames[k])
        for _ in range(args.rounds):
            for k in fps:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    b.track(frames[k])
                fps[k].append(n * args.steps / (time.perf_counter() - t0))
        for k, v in fps.items():
            print(json.dumps({"bench": "sot_track", "config": name, "input": f"{H}x{W}", "frame": f"{h}x{w}", "format": k, "n_seq": n,
                              "frames_per_s": round(max(v), 1), "rounds_frames_per_s": [round(x, 1) for x in v],
                              "h2d_bytes_per_step": n * frames[k][0].numel(), "card": card}), flush=True)
        del b
        torch.cuda.synchronize()


def host(args):
    import cv2
    from unicorn_b200.sot import preprocess
    h, w = 1080, 1920
    nv12 = np.random.default_rng(0).integers(0, 256, (h * 3 // 2, w), dtype=np.uint8)
    out = torch.empty(1, 800, 1280, 3, dtype=torch.uint8)
    ms = []
    for _ in range(args.rounds):
        t0 = time.perf_counter()
        for _ in range(args.steps):
            preprocess(cv2.cvtColor(nv12, cv2.COLOR_YUV2RGB_NV12), (800, 1280), out=out)
        ms.append((time.perf_counter() - t0) * 1e3 / args.steps)
    print(json.dumps({"bench": "host_cpu", "work": "cv2.cvtColor(YUV2RGB_NV12) + sot.preprocess", "frame": f"{h}x{w}", "input": "800x1280",
                      "host_cpu_ms_per_frame": round(min(ms), 2), "rounds_ms": [round(x, 2) for x in ms], "cv2_threads": cv2.getNumThreads(),
                      "host_cpus": os.cpu_count()}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_nv12.py measures on a GPU; none is visible")
    card = gpu_info()
    print(json.dumps({"card": card}), flush=True)
    kernels(args, card)
    sot(args, card)
    host(args)


if __name__ == "__main__":
    main()
