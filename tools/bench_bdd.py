"""The BDD100K test protocol (qdtrack's test_omni.py) batched: UnicornBDDMOTBatch (unicorn_track_large from a *_large_mask state dict,
as the BDD100K recipe loads it) and UnicornBDDMOTSBatch (unicorn_track_large_mask) at n_seq 1 / 2 / 4, 800x1280 from 720x1280 uint8
frames (r = 1), CUDA graphs, seeded weights.

    python tools/bench_bdd.py --workload bdd_mot|bdd_mots [--steps 20] [--n-seq 1 2 4] [--confs 0.01 0.03]

The protocol associates (and for MOTS encodes) every NMS row, and seeded weights leave far more rows than a trained model, so each
line is measured at conf 0.01 (the exp's test_conf) and at a conf that leaves tens of rows per frame.  Printed per line: aggregate
frames/s of pipelined submit(t+1) / collect(t) (host clock around steps that end in a device synchronise), the device step (CUDA
events around graph replays of the step), the mean collect() of a step whose device work is done (association, result assembly and,
for MOTS, every mask's encode), NMS rows and masks encoded per frame.  One JSON line per result."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def frames_720p(n, seed):
    """n seeded 720x1280 uint8 frames letterboxed into 800x1280 (pad 114 below), on the device."""
    from unicorn_b200.synthetic import make_video
    f, _ = make_video(n, 720, 1280, seed=seed, n_obj=6)
    out = torch.full((n, 800, 1280, 3), 114, dtype=torch.uint8)
    out[:, :720] = f.round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1)
    return out.cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=["bdd_mot", "bdd_mots"], default="bdd_mot")
    ap.add_argument("--n-seq", type=int, nargs="+", default=[1, 2, 4])
    ap.add_argument("--confs", type=float, nargs="+", default=[0.01, 0.03])
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    from unicorn_b200.bdd import UnicornBDDMOTBatch, UnicornBDDMOTSBatch
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.weights import load_checkpoint, make_state_dict
    mots = args.workload == "bdd_mots"
    cfg = "unicorn_track_large_mask" if mots else "unicorn_track_large"
    sd = make_state_dict(cfg, 0) if mots else load_checkpoint(make_state_dict("unicorn_track_large_mask", 0), cfg, strict=False)
    eng = UnicornEngine(sd, cfg)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout
    print(json.dumps({"card": torch.cuda.get_device_name(), "nvidia_smi": smi.strip()}), flush=True)
    S = args.steps
    for conf in args.confs:
        for n in args.n_seq:
            cls = UnicornBDDMOTSBatch if mots else UnicornBDDMOTBatch
            trk = cls(eng, (800, 1280), n, conf=conf)
            for i in range(n):
                trk.start(i)
            vid = torch.stack([frames_720p(S + 2, seed=s) for s in range(n)], 1)  # [S+2, n, 800, 1280, 3]
            sizes = [(720, 1280)] * n
            rows = []  # NMS rows of every sequence and frame (host_count, before the max_dets cut)
            for t in range(2):  # eager first step of each parity slot, then its capture
                trk.step_tensor(vid[t], sizes)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            trk.submit(vid[2 % (S + 2)], sizes)
            for t in range(1, S):
                trk.submit(vid[t % (S + 2)], sizes)
                trk.collect()
                rows += [int(v) for v in trk._ctxs[(trk._ring.collected - 1) % 2].host_count]  # the collected step's
            trk.collect()
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            # device step alone: the parity graphs replayed back to back
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for t in range(S):
                trk._ctxs[t % 2].graph.replay()
            ev1.record()
            torch.cuda.synchronize()
            dev_ms = ev0.elapsed_time(ev1) / S
            assoc = []
            for t in range(5):  # collect() of a finished step
                trk.submit(vid[t], sizes)
                torch.cuda.synchronize()
                a0 = time.perf_counter()
                trk.collect()
                assoc.append((time.perf_counter() - a0) * 1e3)
            per_frame = statistics.mean(rows) if rows else 0.0
            print(json.dumps({"workload": args.workload, "config": cfg, "size": [800, 1280], "originals": [[720, 1280]], "driver": cls.__name__,
                              "n_seq": n, "conf": conf, "frames_per_s": round(n * S / wall, 1), "ms_per_step": round(wall * 1e3 / S, 2),
                              "device_ms_per_step": round(dev_ms, 2), "assoc_ms_per_step": round(statistics.median(assoc), 2),
                              "rows_per_frame": round(per_frame, 1), "max_rows_per_frame": max(rows, default=0),
                              "masks_per_frame": round(per_frame, 1) if mots else 0, "max_dets": trk.max_dets,
                              "max_dets_reached": trk._warned, "steps": S}), flush=True)
            del trk, vid
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
