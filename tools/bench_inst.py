"""COCO instance-segmentation throughput and mask output stage on one GPU, seeded weights (unicorn_inst_convnext_tiny).

    python tools/bench_inst.py [--batches 1 8] [--steps 3] [--reps 10] [--stage-only] [--driver-only]

Driver lines: UnicornInstanceSegmenter (CUDA graph per step, chunk 100) at each max_batch, 800x1280 input, synthetic 1080x1920 uint8
frames letterboxed on the device; a step is submit + collect, so it includes every mask chunk, the encodes, the host synchronises and
the string read-back.  images/s = max_batch x steps / s (host clock around whole steps).  Two confidence thresholds: the evaluator's
0.01 (seeded weights leave about 15000 NMS rows per image: 150 chunks) and the conf from a fixed list whose row count is closest to
100 per image.  The mean NMS rows per image are printed with each line.

Stage lines: the mask output stage alone for N = 20 and 100 instances of each of B = 1 and 8 images, 1080x1920 originals, from one
real step's NMS rows, mask features and controller outputs (conf 0.01).  Two arms, each a sequence of launches timed with CUDA events
and alternated in the same process:
  fused: dynamic_masks_rows (d_rate 1, the masks at 400x640) + uc_inst_encode_batched (upsample, resize, threshold, RLE);
  mots:  dynamic_masks at d_rate 2 (fp32 [N, 800, 1280] per image) + uc_mots_encode_batched with one instance per image (so no
         overlap removal, the instance segmentation semantics), in calls of at most 64 instances.
The chars buffers are sized beforehand, so neither arm synchronises.  The strings of both arms are compared (the fused string is
the MOTS one padded to the whole frame).  One JSON line per result, with the card name and power limit read in the same run."""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
NAME, H, W, ORIG = "unicorn_inst_convnext_tiny", 800, 1280, (1080, 1920)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def frames(n, seed=3):
    from unicorn_b200.synthetic import make_video
    f, _ = make_video(n, *ORIG, seed=seed, n_obj=6)
    return [x.permute(1, 2, 0).round().clamp(0, 255).to(torch.uint8).contiguous() for x in f]


def bench_driver(eng, args, info):
    from unicorn_b200.det import UnicornDetector, UnicornInstanceSegmenter
    ims = [t.cuda() for t in frames(max(args.batches))]
    # the conf of the list whose NMS rows per image are closest to 100 on these frames
    rows = {}
    for c in (0.03, 0.04, 0.05, 0.06, 0.08, 0.1, 0.12, 0.15):
        det = UnicornDetector(eng, (H, W), 1, conf=c, use_graph=False)
        rows[c] = sum(det.detect([im])[0][0].shape[0] for im in ims) / len(ims)
    print(json.dumps(dict(nms_rows_per_image_by_conf=rows)), flush=True)
    conf100 = min(rows, key=lambda c: abs(rows[c] - 100))
    for conf in (0.01, conf100):
        for B in args.batches:
            seg = UnicornInstanceSegmenter(eng, (H, W), B, conf=conf)
            step = ims[:B]
            out = seg.detect(step)  # plan-time autotuning, capture
            n_rows = sum(r.shape[0] for r, _, _ in out) / B
            torch.cuda.synchronize()
            times = []
            for _ in range(args.steps):
                t0 = time.perf_counter()
                seg.detect(step)
                times.append(time.perf_counter() - t0)
            med = statistics.median(times)
            print(json.dumps(dict(metric="inst_images_per_s", model=NAME, max_batch=B, conf=conf, nms=0.65, rows_per_image=n_rows,
                                  input=[H, W], orig=list(ORIG), steps=args.steps, step_ms_median=round(med * 1e3, 2),
                                  images_per_s=round(B / med, 3), gpu=info)), flush=True)
            del seg
            torch.cuda.empty_cache()


def bench_stage(eng, args, info):
    from unicorn_b200 import ops, post_ops
    from unicorn_b200.engine import STRIDES
    from unicorn_b200.frames import anchor_count
    from unicorn_b200.results import rle_decode, rle_encode
    h, w, thr = H // 8, W // 8, 0.3
    r = min(H / ORIG[0], W / ORIG[1])
    for B in (1, 8):
        img = torch.stack([ops.letterbox_u8(t.cuda(), (H, W))[0][0] for t in frames(B)])  # [B, H, W, 3] uint8
        ws = ops.PostWorkspace(anchor_count(H, W), "cuda", B)
        eng.begin_frame()
        fpn, _ = eng.backbone(img, tag="stage")
        eng.head(fpn, None, "mot", decode=False, with_masks=True)
        ro, cl, hw = eng.head_maps
        post_ops.det_candidates(ro, cl, hw, STRIDES, 80, 0.01, ws)
        post_ops.postprocess_nms(0.65, ws)
        mf, um = eng.mask_branch(fpn)
        dyn = list(eng.dyn_levels)
        lvl_hw = [(t.shape[1], t.shape[2]) for t in dyn]
        counts = ws.count.tolist()
        image_of = torch.arange(B, dtype=torch.int32, device="cuda")
        for N in (20, 100):
            assert min(counts) >= N, counts
            cnt = torch.full((B,), N, dtype=torch.int32, device="cuda")  # the encode reads the rows [0, N) of each image
            maps = torch.empty(B, N, h * 4, w * 4, device="cuda")
            scratch = torch.empty(B * N * h * w * 17, device="cuda")
            Hs, Ws, rs = [ORIG[0]] * B, [ORIG[1]] * B, [r] * B
            fws = ops.mots_encode_workspace(B * N, *ORIG, "cuda")
            f_emit = torch.empty(B * N, dtype=torch.uint8, device="cuda")
            f_off = torch.empty(B * N + 1, dtype=torch.int64, device="cuda")
            f_chars = torch.empty(64 << 20, dtype=torch.uint8, device="cuda")
            full = torch.empty(B, N, H, W, device="cuda")
            flat = full.view(B * N, 1, H, W)
            nc = (B * N + 63) // 64
            mws = ops.mots_encode_workspace(64, *ORIG, "cuda")
            m_order = torch.zeros(64, dtype=torch.int32, device="cuda")
            m_emit = torch.ones(64, dtype=torch.uint8, device="cuda")
            m_off = torch.empty(nc, 65, dtype=torch.int64, device="cuda")
            m_chars = [torch.empty(16 << 20, dtype=torch.uint8, device="cuda") for _ in range(nc)]

            def fused():
                post_ops.dynamic_masks_rows(mf, um, dyn, lvl_hw, ws.anchors.view(B, -1), cnt, image_of, N, 4, maps, scratch)
                post_ops.inst_encode(maps, cnt, 0, 2, thr, rs, Hs, Ws, fws, f_emit, f_chars, f_off)

            def mots():
                ops.dynamic_masks(mf, um, dyn, lvl_hw, ws, N, up_rate=4, d_rate=2, out=full, scratch=scratch, image_of=image_of)
                for c in range(nc):
                    k = min(64, B * N - 64 * c)
                    ops.mots_encode(flat[64 * c:64 * c + k], m_order[:k], m_emit[:k], thr, [r] * k, [ORIG[0]] * k, [ORIG[1]] * k, mws,
                                    m_chars[c], m_off[c], k=[1] * k)

            arms = dict(fused=fused, mots=mots)
            for fn in arms.values():  # warm-up
                fn()
            torch.cuda.synchronize()
            # both arms give the same masks: every fused string is the MOTS string padded to the whole frame
            fo, mo = f_off.tolist(), m_off.tolist()
            fc, mc = f_chars[:fo[-1]].cpu().numpy().tobytes().decode(), [m_chars[c][:mo[c][min(64, B * N - 64 * c)]].cpu().numpy().tobytes().decode() for c in range(nc)]
            hm, wm = min(ORIG[0], math.floor(H * (1.0 / r))), min(ORIG[1], math.floor(W * (1.0 / r)))
            for j in range(0, B * N, 7):
                s = mc[j // 64][mo[j // 64][j % 64]:mo[j // 64][j % 64 + 1]]
                pad = torch.zeros(ORIG, dtype=torch.bool)
                pad[:hm, :wm] = torch.from_numpy(rle_decode(s, hm, wm))
                assert fc[fo[j]:fo[j + 1]] == rle_encode(pad.numpy()), (B, N, j)
            ms = {k: [] for k in arms}
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            for _ in range(args.reps):
                for k, fn in arms.items():
                    ev[0].record()
                    fn()
                    ev[1].record()
                    ev[1].synchronize()
                    ms[k].append(ev[0].elapsed_time(ev[1]))
            full_bytes = B * N * H * W * 4
            print(json.dumps(dict(metric="inst_mask_stage_ms", B=B, N=N, orig=list(ORIG), input=[H, W], reps=args.reps,
                                  fused_ms_median=round(statistics.median(ms["fused"]), 3), mots_ms_median=round(statistics.median(ms["mots"]), 3),
                                  fused_ms_min=round(min(ms["fused"]), 3), mots_ms_min=round(min(ms["mots"]), 3),
                                  full_res_mask_bytes_written_by_mots_arm=full_bytes, gpu=info)), flush=True)
            del maps, scratch, full, flat, m_chars, f_chars
            torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 8])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--stage-only", action="store_true")
    ap.add_argument("--driver-only", action="store_true")
    args = ap.parse_args()
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import make_state_dict
    info = gpu_info()
    print(json.dumps(dict(gpu=info)), flush=True)
    eng = UnicornEngine(make_state_dict(NAME, 0), NAME)
    if not args.driver_only:
        bench_stage(eng, args, info)
    if not args.stage_only:
        bench_driver(eng, args, info)


if __name__ == "__main__":
    main()
