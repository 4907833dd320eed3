"""COCO detector throughput and post-processing time on one GPU, seeded weights, CUDA graphs.

    python tools/bench_det.py [--models unicorn_det_convnext_tiny ...] [--batches 1 8 32] [--steps 20] [--rounds 3] [--post-only]

Detector lines: UnicornDetector at each max_batch, 800x1280 input, images already letterboxed in HBM: a step is a replay of the
step's graph (backbone, neck, head, fused candidates, sort, NMS), timed with CUDA events; images/s = max_batch x steps / s.  Every
detector of a model is built first (plan-time autotuning, capture); the timed rounds then alternate over them.

Post-processing lines (--post-only runs just these): the 80-class head maps of B images at 800x1280 (random logits, about a third
of the anchors above conf 0.01), four arms captured as CUDA graphs and timed alternately: head_decode + postprocess (decode, filter,
sort, NMS), the fused det_candidates + the same sort and NMS, head_decode alone and det_candidates alone.  The old filter has no entry
point of its own; since both pipelines hand bit-identical candidates to the same sort and NMS, its time with the decode is the fused
arm's plus the difference of the two full pipelines.  One JSON line per result, with the card name, power limit and SM clock read in the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def graph_of(fn, reps=1):
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    g.replay()
    torch.cuda.synchronize()
    return g


def time_graph(g, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def bench_post(args, info):
    from unicorn_b200 import ops, post_ops
    from unicorn_b200.engine import STRIDES
    H, W, ncls = 800, 1280, 80
    for B in (1, 32):
        g = torch.Generator(device="cuda").manual_seed(B)
        ro, cl, hw = [], [], []
        for s in STRIDES:
            h, w = H // s, W // s
            r = torch.randn(B, h, w, 8, device="cuda", generator=g) * 0.5
            r[..., 4] = torch.randn(B, h, w, device="cuda", generator=g) - 1.0
            ro.append(r)
            cl.append(torch.randn(B, h, w, ncls, device="cuda", generator=g) - 6.0)
            hw.append((h, w))
        A = sum(h * w for h, w in hw)
        ws = ops.PostWorkspace(A, "cuda", B)
        pred = torch.empty(B, A, 5 + ncls, device="cuda")

        def decode_filter():
            ops.head_decode(ro, cl, hw, STRIDES, ncls, out=pred if B > 1 else pred[0])
            ops.postprocess_device(pred, ncls, 0.01, 0.65, ws)

        def fused(nms=True):
            post_ops.det_candidates(ro, cl, hw, STRIDES, ncls, 0.01, ws)
            if nms:
                post_ops.postprocess_nms(0.65, ws)
        arms = {"decode+filter+sort+nms": graph_of(decode_filter), "fused+sort+nms": graph_of(fused),
                "head_decode": graph_of(lambda: ops.head_decode(ro, cl, hw, STRIDES, ncls, out=pred if B > 1 else pred[0])),
                "fused": graph_of(lambda: fused(False))}
        cands = [int(c) for c in ws.count.tolist()]
        times = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, gr in arms.items():
                time_graph(gr, 20)
                times[k].append(time_graph(gr, 200) * 1e3)
        print(json.dumps(dict(kind="post", B=B, A=A, ncls=ncls, candidates_per_image=round(sum(cands) / len(cands)), gpu=info,
                              us={k: round(statistics.median(v), 1) for k, v in times.items()},
                              us_all={k: [round(x, 1) for x in v] for k, v in times.items()})), flush=True)


def bench_models(args, info):
    from unicorn_b200.det import UnicornDetector
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.weights import make_state_dict
    H, W = 800, 1280
    frames, _ = make_video(2, H, W, seed=1, n_obj=5)
    img = frames[1].permute(1, 2, 0).clamp(0, 255).to(torch.uint8).contiguous()
    for name in args.models:
        eng = UnicornEngine(make_state_dict(name, 0), name)
        dets = {}
        for B in args.batches:
            d = UnicornDetector(eng, (H, W), max_batch=B)
            rows = d.detect([img.numpy()] * B)
            dets[B] = (d, sum(r.shape[0] for r, _ in rows) / B)
        times = {B: [] for B in dets}
        for _ in range(args.rounds):
            for B, (d, _) in dets.items():
                c = d._ring.slots[0]
                time_graph(c.graph, 3)
                times[B].append(time_graph(c.graph, args.steps))
        for B, (d, nrow) in dets.items():
            ms = statistics.median(times[B])
            print(json.dumps(dict(kind="detector", model=name, max_batch=B, input=[H, W], ms_per_step=round(ms, 3),
                                  images_per_s=round(B * 1e3 / ms, 1), ms_all=[round(x, 3) for x in times[B]], rows_per_image=nrow,
                                  launches_per_step=d.launches_per_step, gpu=info)), flush=True)
        del dets, eng
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", nargs="+", default=["unicorn_det_convnext_tiny", "unicorn_det_r50", "unicorn_det_convnext_large"])
    ap.add_argument("--batches", nargs="+", type=int, default=[1, 8, 32])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--post-only", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_det: needs a CUDA GPU")
    info = gpu_info()
    bench_post(args, info)
    if not args.post_only:
        bench_models(args, info)


if __name__ == "__main__":
    main()
