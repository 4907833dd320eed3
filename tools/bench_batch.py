"""Several SOT sequences per GPU: one batched frame (UnicornSOTBatch, n_seq sequences in lock step) against frames in flight of one
sequence (UnicornSOTTrack, depth 1 and 3), on the 800x1280 SOT frame with CUDA graphs.

    python tools/bench_batch.py [--steps 60] [--rounds 3] [--configs unicorn_track_large unicorn_track_r50] [--n-seq 1 2 4 8]

--workload vos: the same for VOS with 1 and 3 objects per sequence (--objects): UnicornVOSBatch at n_seq 1 / 2 / 4 against
UnicornVOSTrack at depth 1 and 3, unicorn_track_large_mask by default.  A VOS step is timed end to end (host clock around steps that
end in a device synchronise): input copy, graph replay, the read-back of the detection rows and the per-sequence result assembly.

--workload mot: UnicornMOTBatch at n_seq 1 / 2 / 4 against UnicornMOTTracker(use_graph=True) driven with pipelined submit / collect, QD
arm, unicorn_track_large; --assoc byte: the ByteTrack arm, against UnicornMOTTracker(assoc="byte") at depth 1 and 3.  A step is timed
end to end (host clock around steps that end in a device synchronise, the association included).  Also printed: the device-only step
(CUDA events around graph replays of the step), the mean host association per step (collect() of a step whose device work is done),
the mean detections handed to the trackers per frame and the kernels launched per step.

--workload mots: UnicornMOTSBatch at n_seq 1 / 2 / 4 against UnicornMOTSTracker(use_graph=True) driven with pipelined submit / collect,
unicorn_track_large_mot_challenge_mask, the sequences' frames letterboxed from 1080x1920 and 480x640 originals in turn.  The same
fields as the mot lines, plus each parity slot's mask buffer (n_seq x max_dets x H x W fp32).  Seeded weights leave no track at the
default score_thr = 0.1, so these lines measure the frame; the encode-alone line measures the encoder: n_seq sequences of 20 synthetic
instances each (1080x1920 and 480x640 originals in turn), one MaskEncoder.batch call against n_seq one-frame MaskEncoder calls, each
timed with CUDA events around the whole call (its host synchronises included).

Device-resident timing like bench.py's `value`: the frames are already in HBM, each step is an input copy and a graph replay, timed
with CUDA events.  Every driver of a config is built first (plan-time autotuning of the batched layer shapes, graph capture); the
timed rounds then alternate over the drivers so that clock and neighbour drift spread over all of them.  Printed per driver: aggregate
frames/s (sequences x steps / s), ms per step, and the device memory the driver added on top of what was already allocated (the
engine's weights and the drivers built before it): the peak torch allocation while it was built and warmed up, minus the allocation
before.  One JSON line per result."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=["sot", "vos", "mot", "mots"], default="sot")
    ap.add_argument("--assoc", choices=["qd", "byte"], default="qd")
    ap.add_argument("--n-obj", type=int, default=6)
    ap.add_argument("--configs", nargs="+", default=None)
    ap.add_argument("--size", type=int, nargs=2, default=(800, 1280))
    ap.add_argument("--n-seq", type=int, nargs="+", default=None)
    ap.add_argument("--objects", type=int, nargs="+", default=[1, 3])
    ap.add_argument("--depths", type=int, nargs="+", default=[1, 3])
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if args.workload == "vos":
        args.configs = args.configs or ["unicorn_track_large_mask"]
        args.n_seq = args.n_seq or [1, 2, 4]
        return main_vos(args)
    if args.workload == "mot":
        args.configs = args.configs or ["unicorn_track_large"]
        args.n_seq = args.n_seq or [1, 2, 4]
        return main_mot(args)
    if args.workload == "mots":
        args.configs = args.configs or ["unicorn_track_large_mot_challenge_mask"]
        args.n_seq = args.n_seq or [1, 2, 4]
        return main_mots(args)
    args.configs = args.configs or ["unicorn_track_large", "unicorn_track_r50"]
    args.n_seq = args.n_seq or [1, 2, 4, 8]
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.sot import UnicornSOTBatch, UnicornSOTTrack
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.weights import make_state_dict

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": torch.cuda.get_device_name(), "nvidia_smi": q}), flush=True)
    H, W = args.size
    N = max(args.n_seq)
    to_u8 = lambda f: f.round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()  # noqa: E731
    main_stream = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for cfg in args.configs:
        eng = UnicornEngine(make_state_dict(cfg, 0), cfg)
        videos = [make_video(5, H, W, seed=s) for s in range(N)]
        refs = [(to_u8(fr[0:1]), bx[0, 0]) for fr, bx in videos]
        steps_u8 = [torch.stack([to_u8(fr[1 + t:2 + t])[0] for fr, _ in videos]).cuda() for t in range(4)]  # [N,H,W,3] per step
        drivers = {}
        for n in args.n_seq:
            m0 = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            sb = UnicornSOTBatch(eng, (H, W), n)
            for i in range(n):
                sb.initialize_tensor(i, *refs[i])
            for t in range(3):
                sb.track_tensor(steps_u8[t][:n])

            def batch_step(t, sb=sb, n=n):
                sb.slot.img_in_u8.copy_(steps_u8[t % 4][:n], non_blocking=True)
                sb.slot.graph.replay()
            drivers[f"batch{n}"] = (batch_step, n, [], torch.cuda.max_memory_allocated() - m0)
        for d in args.depths:
            m0 = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            trk = UnicornSOTTrack(eng, (H, W), depth=d)
            trk.initialize_tensor(*refs[0])
            for t in range(2 * d + 1):
                trk.track_tensor(steps_u8[t % 4][0:1])

            def pipe_step(t, trk=trk, d=d):
                c = trk._ctxs[t % d]
                with torch.cuda.stream(c.stream):
                    c.img_in_u8.copy_(steps_u8[t % 4][0:1], non_blocking=True)
                    c.graph.replay()
            drivers[f"depth{d}"] = (pipe_step, 1, [c.stream for c in trk._ctxs if c.stream is not None], torch.cuda.max_memory_allocated() - m0)
        times = {k: [] for k in drivers}
        for _ in range(args.rounds):
            for k, (step, n, streams, _) in drivers.items():
                torch.cuda.synchronize()
                e0.record()
                for st in streams:  # frames in flight: fork from the timed region's start, join before its end
                    st.wait_stream(main_stream)
                for t in range(args.steps):
                    step(t)
                for st in streams:
                    main_stream.wait_stream(st)
                e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1) / 1e3)
        for k, (step, n, streams, mem) in drivers.items():
            ts = times[k]
            fps = [n * args.steps / t for t in ts]
            print(json.dumps({"config": cfg, "size": [H, W], "driver": "UnicornSOTBatch" if k.startswith("batch") else "UnicornSOTTrack",
                              "n_seq": n, "depth": max(1, len(streams)), "frames_per_s": round(statistics.median(fps), 1),
                              "frames_per_s_min_max": [round(min(fps), 1), round(max(fps), 1)],
                              "ms_per_step": round(1e3 * statistics.median(ts) / args.steps, 2),
                              "added_peak_alloc_gib": round(mem / 2 ** 30, 2), "steps": args.steps, "rounds": args.rounds}), flush=True)
        del drivers, eng, sb, trk, batch_step, pipe_step
        torch.cuda.empty_cache()


def main_vos(args):
    import time
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.vos import UnicornVOSBatch, UnicornVOSTrack
    from unicorn_b200.weights import make_state_dict

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": torch.cuda.get_device_name(), "nvidia_smi": q}), flush=True)
    H, W = args.size
    N = max(args.n_seq)
    to_u8 = lambda f: f.round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()  # noqa: E731
    for cfg in args.configs:
        eng = UnicornEngine(make_state_dict(cfg, 0), cfg)
        for k in args.objects:
            videos = [make_video(5, H, W, seed=s, n_obj=k) for s in range(N)]
            refs = [(to_u8(fr[0:1]).cuda(), {o + 1: bx[0, o] for o in range(k)}) for fr, bx in videos]
            steps_u8 = [torch.stack([to_u8(fr[1 + t:2 + t])[0] for fr, _ in videos]).cuda() for t in range(4)]  # [N,H,W,3] per step
            drivers = {}
            for n in args.n_seq:
                m0 = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                vb = UnicornVOSBatch(eng, (H, W), n, max_objects=n * k, max_groups=n * -(-k // 8))
                for i in range(n):
                    vb.initialize_tensor(i, *refs[i])
                for t in range(3):
                    vb.track_tensor(steps_u8[t][:n])

                def batch_round(steps, vb=vb, n=n):
                    for t in range(steps):
                        vb.track_tensor(steps_u8[t % 4][:n])
                drivers[f"batch{n}"] = ("UnicornVOSBatch", batch_round, n, 1, torch.cuda.max_memory_allocated() - m0, vb)
            for d in args.depths:
                m0 = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                trk = UnicornVOSTrack(eng, (H, W), use_graph=True, depth=d)
                trk.initialize_tensor(*refs[0])
                for t in range(2 * d + 1):
                    trk.track_tensor(steps_u8[t % 4][0:1])

                def pipe_round(steps, trk=trk, d=d):
                    sub = 0
                    for c in range(steps):
                        while sub < steps and sub - c < d:
                            trk.submit(steps_u8[sub % 4][0:1])
                            sub += 1
                        trk.collect()
                drivers[f"depth{d}"] = ("UnicornVOSTrack", pipe_round, 1, d, torch.cuda.max_memory_allocated() - m0, trk)
            times = {key: [] for key in drivers}
            for _ in range(args.rounds):
                for key, (_, run, _, _, _, _) in drivers.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    run(args.steps)
                    torch.cuda.synchronize()
                    times[key].append(time.perf_counter() - t0)
            for key, (name, _, n, d, mem, drv) in drivers.items():
                ts = times[key]
                fps = [n * args.steps / t for t in ts]
                print(json.dumps({"workload": "vos", "config": cfg, "size": [H, W], "objects_per_seq": k, "driver": name, "n_seq": n, "depth": d,
                                  "frames_per_s": round(statistics.median(fps), 1), "frames_per_s_min_max": [round(min(fps), 1), round(max(fps), 1)],
                                  "ms_per_step": round(1e3 * statistics.median(ts) / args.steps, 2),
                                  "launches_per_step": drv.launches_per_frame,
                                  "added_peak_alloc_gib": round(mem / 2 ** 30, 2), "steps": args.steps, "rounds": args.rounds}), flush=True)
            del drivers, vb, trk, drv, batch_round, pipe_round
            torch.cuda.empty_cache()


class _Counting:
    """Forwards to a tracker and counts the detections handed to it (QD: the boxes passed to match, ByteTrack: the rows passed to
    update)."""

    def __init__(self, trk):
        self.trk, self.dets, self.calls = trk, 0, 0

    def match(self, boxes, *a, **kw):
        self.dets, self.calls = self.dets + boxes.shape[0], self.calls + 1
        return self.trk.match(boxes, *a, **kw)

    def update(self, dets, *a, **kw):
        self.dets, self.calls = self.dets + dets.shape[0], self.calls + 1
        return self.trk.update(dets, *a, **kw)

    def __getattr__(self, name):
        return getattr(self.trk, name)


def main_mot(args):
    import time
    import types
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.mot import UnicornMOTBatch, UnicornMOTTracker
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    from unicorn_b200.tracker.byte_tracker import BYTETracker
    from unicorn_b200.weights import make_state_dict

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": torch.cuda.get_device_name(), "nvidia_smi": q}), flush=True)
    H, W = args.size
    N = max(args.n_seq)
    to_u8 = lambda f: f.round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()  # noqa: E731
    bargs = types.SimpleNamespace(track_thresh=0.5, track_buffer=30, match_thresh=0.8, mot20=False)
    new_tracker = lambda: _Counting(QuasiDenseEmbedTracker() if args.assoc == "qd" else BYTETracker(bargs))  # noqa: E731
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for cfg in args.configs:
        eng = UnicornEngine(make_state_dict(cfg, 0), cfg)
        videos = [make_video(4, H, W, seed=s, n_obj=args.n_obj)[0] for s in range(N)]
        steps_u8 = [torch.stack([to_u8(v[t:t + 1])[0] for v in videos]).cuda() for t in range(4)]  # [N,H,W,3] per step
        drivers = {}
        for n in args.n_seq:
            m0 = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            mb = UnicornMOTBatch(eng, (H, W), n, assoc=args.assoc, use_graph=True)
            trackers = [new_tracker() for _ in range(n)]
            for i in range(n):
                mb.start(i, trackers[i])

            def batch_round(steps, mb=mb, n=n):  # submit(t+1) before collect(t)
                mb.submit(steps_u8[0][:n])
                for t in range(steps):
                    if t + 1 < steps:
                        mb.submit(steps_u8[(t + 1) % 4][:n])
                    mb.collect()

            def batch_assoc(t, mb=mb, n=n):
                mb.submit(steps_u8[t % 4][:n])
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                mb.collect()
                return time.perf_counter() - t0

            def batch_replay(t, mb=mb, n=n):
                c = mb._ctxs[t % 2]
                c.img_in_u8.copy_(steps_u8[t % 4][:n], non_blocking=True)
                c.graph.replay()
            batch_round(4)
            drivers[f"batch{n}"] = ("UnicornMOTBatch", batch_round, batch_assoc, batch_replay, n, 1, mb, mb.launches_per_frame, trackers,
                                    torch.cuda.max_memory_allocated() - m0)
        for d in ([1] if args.assoc == "qd" else args.depths):
            m0 = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            trk = UnicornMOTTracker(eng, (H, W), assoc=args.assoc, tracker=new_tracker(), use_graph=True, depth=d)
            trk.step_tensor(steps_u8[0][0:1], img_info=(H, W))
            l0 = _launches()
            trk.submit(steps_u8[1][0:1])  # a slot's first frame runs eagerly: its launches are every frame's device half
            launches = _launches() - l0
            trk.collect((H, W))
            inflight = max(2, d)  # depth 1: the two parity slots let submit(t+1) precede collect(t)

            def pipe_round(steps, trk=trk, k=inflight):
                sub = 0
                for c in range(steps):
                    while sub < steps and sub - c < k:
                        trk.submit(steps_u8[sub % 4][0:1])
                        sub += 1
                    trk.collect((H, W))

            def pipe_assoc(t, trk=trk):
                trk.submit(steps_u8[t % 4][0:1])
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                trk.collect((H, W))
                return time.perf_counter() - t0

            def pipe_replay(t, trk=trk):
                c = trk._ctxs[t % len(trk._ctxs)]
                with torch.cuda.stream(c.stream):
                    c.img_in_u8.copy_(steps_u8[t % 4][0:1], non_blocking=True)
                    c.graph.replay()
            pipe_round(4 + 2 * d)
            drivers[f"depth{d}"] = ("UnicornMOTTracker", pipe_round, pipe_assoc, pipe_replay, 1, d, trk, launches, [trk.tracker],
                                    torch.cuda.max_memory_allocated() - m0)
        times = {key: [] for key in drivers}
        for _ in range(args.rounds):
            for key, (_, run, *_rest) in drivers.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                run(args.steps)
                torch.cuda.synchronize()
                times[key].append(time.perf_counter() - t0)
        main_stream = torch.cuda.current_stream()
        for key, (name, _, assoc, replay, n, d, drv, launches, trackers, mem) in drivers.items():
            for t in trackers:
                t.dets = t.calls = 0
            a = [assoc(t) for t in range(10)]
            frames = sum(t.calls for t in trackers)
            streams = [c.stream for c in drv._ctxs if c.stream is not None]
            torch.cuda.synchronize()
            e0.record()
            for st in streams:
                st.wait_stream(main_stream)
            for t in range(args.steps):
                replay(t)
            for st in streams:
                main_stream.wait_stream(st)
            e1.record()
            torch.cuda.synchronize()
            ts = times[key]
            fps = [n * args.steps / t for t in ts]
            print(json.dumps({"workload": "mot", "assoc": args.assoc, "config": cfg, "size": [H, W], "driver": name, "n_seq": n, "depth": d,
                              "frames_per_s": round(statistics.median(fps), 1), "frames_per_s_min_max": [round(min(fps), 1), round(max(fps), 1)],
                              "ms_per_step": round(1e3 * statistics.median(ts) / args.steps, 2),
                              "device_ms_per_step": round(e0.elapsed_time(e1) / args.steps, 2),
                              "assoc_ms_per_step": round(1e3 * statistics.mean(a), 2),
                              "dets_per_frame": round(sum(t.dets for t in trackers) / max(frames, 1), 1),
                              "launches_per_step": launches,
                              "added_peak_alloc_gib": round(mem / 2 ** 30, 2), "steps": args.steps, "rounds": args.rounds}), flush=True)
        del drivers, drv, trackers, eng
        torch.cuda.empty_cache()


def _blobs(n, H, W, seed):
    """n synthetic 0 / 1 instance masks [n, H, W] on the device: ellipses of random centre and axes."""
    g = torch.Generator().manual_seed(seed)
    c = torch.rand(n, 2, generator=g) * torch.tensor([H, W])
    a = 30 + torch.rand(n, 2, generator=g) * torch.tensor([H / 4, W / 4])
    yy, xx = torch.arange(H, device="cuda", dtype=torch.float32), torch.arange(W, device="cuda", dtype=torch.float32)
    c, a = c.cuda(), a.cuda()
    return ((((yy[None, :, None] - c[:, 0, None, None]) / a[:, 0, None, None]) ** 2 +
             ((xx[None, None, :] - c[:, 1, None, None]) / a[:, 1, None, None]) ** 2) < 1).float()


def main_mots(args):
    import time
    from unicorn_b200 import ops
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.mots import MaskEncoder, UnicornMOTSBatch, UnicornMOTSTracker
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.weights import make_state_dict

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": torch.cuda.get_device_name(), "nvidia_smi": q}), flush=True)
    H, W = args.size
    N = max(args.n_seq)
    origs = [(1080, 1920), (480, 640)]  # sequence i comes from origs[i % 2]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for cfg in args.configs:
        eng = UnicornEngine(make_state_dict(cfg, 0), cfg)
        seqs = []
        for s in range(N):
            h, w = origs[s % 2]
            raw = make_video(4, h, w, seed=s, n_obj=args.n_obj)[0].round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous().cuda()
            seqs.append(torch.cat([ops.letterbox_u8(raw[t], (H, W), swap_rb=False)[0] for t in range(4)]))
        steps_u8 = [torch.stack([v[t] for v in seqs]) for t in range(4)]  # [N,H,W,3] per step
        sizes = [origs[s % 2] for s in range(N)]
        drivers = {}
        for n in args.n_seq:
            m0 = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            mb = UnicornMOTSBatch(eng, (H, W), n, use_graph=True)
            for i in range(n):
                mb.start(i)

            def batch_round(steps, mb=mb, n=n):  # submit(t+1) before collect(t)
                mb.submit(steps_u8[0][:n], sizes[:n])
                for t in range(steps):
                    if t + 1 < steps:
                        mb.submit(steps_u8[(t + 1) % 4][:n], sizes[:n])
                    mb.collect()

            def batch_assoc(t, mb=mb, n=n):
                mb.submit(steps_u8[t % 4][:n], sizes[:n])
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                mb.collect()
                return time.perf_counter() - t0

            def batch_replay(t, mb=mb, n=n):
                c = mb._ctxs[t % 2]
                c.img_in_u8.copy_(steps_u8[t % 4][:n], non_blocking=True)
                c.graph.replay()
            batch_round(4)
            drivers[f"batch{n}"] = ("UnicornMOTSBatch", batch_round, batch_assoc, batch_replay, n, mb.launches_per_frame, mb.max_dets,
                                    torch.cuda.max_memory_allocated() - m0)
        m0 = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        trk = UnicornMOTSTracker(eng, (H, W), use_graph=True)
        trk.step_tensor(steps_u8[0][0:1], *sizes[0])
        l0 = _launches()
        trk.submit(steps_u8[1][0:1], *sizes[0])  # a slot's first frame runs eagerly: its launches are every frame's device half
        launches = _launches() - l0
        trk.collect()

        def pipe_round(steps, trk=trk):
            trk.submit(steps_u8[0][0:1], *sizes[0])
            for t in range(steps):
                if t + 1 < steps:
                    trk.submit(steps_u8[(t + 1) % 4][0:1], *sizes[0])
                trk.collect()

        def pipe_assoc(t, trk=trk):
            trk.submit(steps_u8[t % 4][0:1], *sizes[0])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            trk.collect()
            return time.perf_counter() - t0

        def pipe_replay(t, trk=trk):
            c = trk._ctxs[t % 2]
            c.img_in_u8.copy_(steps_u8[t % 4][0:1], non_blocking=True)
            c.graph.replay()
        pipe_round(4)
        drivers["depth1"] = ("UnicornMOTSTracker", pipe_round, pipe_assoc, pipe_replay, 1, launches, trk.max_dets,
                             torch.cuda.max_memory_allocated() - m0)
        times = {key: [] for key in drivers}
        for _ in range(args.rounds):
            for key, (_, run, *_rest) in drivers.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                run(args.steps)
                torch.cuda.synchronize()
                times[key].append(time.perf_counter() - t0)
        for key, (name, _, assoc, replay, n, launches, max_dets, mem) in drivers.items():
            a = [assoc(t) for t in range(10)]
            torch.cuda.synchronize()
            e0.record()
            for t in range(args.steps):
                replay(t)
            e1.record()
            torch.cuda.synchronize()
            ts = times[key]
            fps = [n * args.steps / t for t in ts]
            print(json.dumps({"workload": "mots", "config": cfg, "size": [H, W], "originals": sizes[:n], "driver": name, "n_seq": n,
                              "frames_per_s": round(statistics.median(fps), 1), "frames_per_s_min_max": [round(min(fps), 1), round(max(fps), 1)],
                              "ms_per_step": round(1e3 * statistics.median(ts) / args.steps, 2),
                              "device_ms_per_step": round(e0.elapsed_time(e1) / args.steps, 2),
                              "assoc_ms_per_step": round(1e3 * statistics.mean(a), 2), "launches_per_step": launches,
                              "mask_buffer_gib_per_slot": round(n * max_dets * H * W * 4 / 2 ** 30, 3),
                              "added_peak_alloc_gib": round(mem / 2 ** 30, 2), "steps": args.steps, "rounds": args.rounds}), flush=True)
        del drivers, trk, eng
        torch.cuda.empty_cache()
    # the encoder alone: n_seq sequences of 20 tracked instances each
    k, reps = 20, 20
    for n in args.n_seq:
        masks = torch.stack([_blobs(64, H, W, s) for s in range(n)])
        frames = []
        for s in range(n):
            g = torch.Generator().manual_seed(100 + s)
            h, w = origs[s % 2]
            frames.append((torch.randperm(64, generator=g)[:k].tolist(), [i % 5 != 4 for i in range(k)], min(H / h, W / w), h, w))
        batch_enc, one_enc = MaskEncoder(n * 64, "cuda"), MaskEncoder(64, "cuda")
        run_batch = lambda: batch_enc.batch(masks, 0.3, frames)  # noqa: E731
        run_loop = lambda: [one_enc(masks[s], *frames[s][:2], 0.3, *frames[s][2:]) for s in range(n)]  # noqa: E731
        same = run_batch() == run_loop()  # also the warm-up (workspaces, buffer growth)
        ms, launches = {}, {}
        for _ in range(3):  # alternate the two
            for key, fn in (("batched", run_batch), ("loop", run_loop)):
                l0 = _launches()
                t = []
                for _ in range(reps):
                    e0.record()
                    fn()
                    e1.record()
                    e1.synchronize()
                    t.append(e0.elapsed_time(e1))
                ms.setdefault(key, []).extend(t)
                launches[key] = (_launches() - l0) // reps
        print(json.dumps({"workload": "mots_encode", "size": [H, W], "n_seq": n, "instances_per_seq": k, "originals": [f[3:] for f in frames],
                          "batched_ms": round(statistics.median(ms["batched"]), 3), "loop_ms": round(statistics.median(ms["loop"]), 3),
                          "batched_ms_min_max": [round(min(ms["batched"]), 3), round(max(ms["batched"]), 3)],
                          "loop_ms_min_max": [round(min(ms["loop"]), 3), round(max(ms["loop"]), 3)],
                          "launches": launches, "identical_strings": same}), flush=True)
        del masks


def _launches():
    from unicorn_b200 import _lib
    return _lib.LAUNCHES


if __name__ == "__main__":
    main()
