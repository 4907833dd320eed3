"""BDD100K MOTS bitmasks: the host restatement of qdtrack's mask_prepare + mask_merge (oracle/bdd_bitmask_oracle.py) against the device
painter (unicorn_b200.bdd.BDDBitmasks.paint) at 720 x 1280, K tracked instances per frame and B frames per call, and PIL's PNG write
of the same bitmasks on its own (what write_seg_track leaves on the host).

    python tools/bench_bdd_bitmask.py [--reps 20] [--oracle-reps 1]

The painter's time is wall time per call from the track_result dicts to the bitmasks in pinned host memory: host packing, the string
upload, the launches and the readback, ended by the synchronise paint() does.  Each configuration's bitmasks are checked against the
oracle byte for byte.  Prints the card and its power limit, one line per configuration and a JSON summary line."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import bdd_bitmask_oracle as bo  # noqa: E402
from unicorn_b200.bdd import BDDBitmasks  # noqa: E402
from unicorn_b200.results import rle_dict, rle_encode  # noqa: E402

H, W = 720, 1280


def frame(rng, k):
    """k tracked instances: ellipses of 20..300 x 20..400 pixels (BDD100K's cars and pedestrians), distinct scores, labels 0..7."""
    yy, xx = np.mgrid[:H, :W]
    d = {}
    for n, s in enumerate(rng.permutation(1 << 16)[:k]):
        cy, cx, ry, rx = rng.integers(0, H), rng.integers(0, W), rng.integers(10, 150), rng.integers(10, 200)
        m = ((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 <= 1.0
        d[np.int64(rng.integers(0, 1 << 17))] = dict(bbox=np.array([0, 0, 1, 1, s / 65536], dtype=np.float32), label=np.float32(n % 8),
                                                     segm=rle_dict(rle_encode(m), H, W))
    return d


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--oracle-reps", type=int, default=1)
    ap.add_argument("--ks", default="10,30,100")
    ap.add_argument("--bs", default="1,8")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bdd_bitmask: no GPU")
    gpu = card()
    print("card, power limit:", gpu)
    painter = BDDBitmasks("cuda")
    rng = np.random.default_rng(0)
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        from PIL import Image
        for k in [int(v) for v in a.ks.split(",")]:
            for B in [int(v) for v in a.bs.split(",")]:
                frames = [frame(rng, k) for _ in range(B)]
                sizes = [(H, W)] * B
                t0 = time.perf_counter()
                for _ in range(a.oracle_reps):
                    want = [bo.bdd_bitmask(d, H, W) for d in frames]
                t_oracle = (time.perf_counter() - t0) / a.oracle_reps
                for _ in range(3):
                    got = painter.paint(frames, sizes, host=True)
                assert all(np.array_equal(x, y) for x, y in zip(got, want)), (k, B)
                ts = []
                for _ in range(a.reps):
                    t0 = time.perf_counter()
                    painter.paint(frames, sizes, host=True)
                    ts.append(time.perf_counter() - t0)
                t_dev = float(np.median(ts))
                t0 = time.perf_counter()
                for i, bm in enumerate(want):
                    Image.fromarray(bm).save(os.path.join(tmp, f"{k}_{B}_{i}.png"))
                t_png = (time.perf_counter() - t0) / B
                row = dict(k=k, B=B, oracle_ms_per_frame=1e3 * t_oracle / B, paint_ms_per_call=1e3 * t_dev, paint_ms_per_frame=1e3 * t_dev / B,
                           paint_min_ms_per_call=1e3 * min(ts), png_write_ms_per_frame=1e3 * t_png, speedup=t_oracle / t_dev,
                           chars=sum(len(v["segm"]["counts"]) for d in frames for v in d.values()))
                rows.append(row)
                print(f"K={k:4d} B={B:2d}  oracle {row['oracle_ms_per_frame']:9.2f} ms/frame  paint {row['paint_ms_per_call']:7.3f} ms/call "
                      f"({row['paint_ms_per_frame']:6.3f} ms/frame, min {row['paint_min_ms_per_call']:.3f})  x{row['speedup']:8.1f}  "
                      f"PNG write {row['png_write_ms_per_frame']:6.2f} ms/frame", flush=True)
    print(json.dumps(dict(metric="bdd_bitmask", card=gpu, frame=[H, W], rows=rows)))


if __name__ == "__main__":
    main()
