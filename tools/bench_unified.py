"""SOT targets plus a MOT arm on one video: UnicornUnifiedTracker (one backbone pass per frame) against the same work done by today's
two drivers in the same process, UnicornSOTBatch(n_seq=K) fed K copies of the frame plus UnicornMOTTracker.

    python tools/bench_unified.py [--configs unicorn_track_large unicorn_track_r50] [--targets 1 2 4] [--mot qd byte none] [--steps 20]

800x1280, seeded weights, make_video(..., n_obj=6) frames resident on the device as uint8, CUDA graphs everywhere.  K targets are
added on frame 0, one per object.  Both sides run the MOT driver's protocol (submit(t + 1) before collect(t), the association
included); the two-driver side collects the SOT batch of step t before submitting its next one.  A step is timed end to end: host
clock around `steps` steps that end in a device synchronise, three rounds alternating between the two sides; median and min-max.
Also printed: the device-only step (CUDA events around graph replays of the step with its input copy), the kernels launched per
step through the C ABI, and the device memory each side added on top of what was already allocated (peak allocation while it was
built and warmed up, minus the allocation before).  The card's name and power limit are printed first.  One JSON line per
(config, K, mot).

    python tools/bench_unified.py --workload mask [--configs ...] [--objects 1 3] [--mots on off] [--steps 20]

The mask workload: VOS objects plus a MOTS arm on one video, UnicornUnifiedMaskTracker against UnicornVOSTrack(use_graph=True,
depth=2) plus UnicornMOTSTracker(use_graph=True), both pipelined (submit(t + 1) before collect(t)), on unicorn_track_large_mask and
unicorn_track_large_mot_challenge_mask.  The video is 1080x1920: its frames are letterboxed once on the host to 800x1280 uint8 and kept
on the device, and the label map, soft masks and MOTS strings are produced at 1080x1920.  The objects are added on frame 0, in one
group.  A step includes the VOS result assembly, the MOTS association and the mask encode.  The device-only step is the graph
replays with their input copies, plus the unified tracker's result assembly, which runs after its graph (UnicornVOSTrack captures
its own).  Launches per step count the kernels of the graphs plus the launches outside them (assembly, encode).  One JSON line per
(config, objects, mots).

    python tools/bench_unified.py --workload batch [--configs ...] [--n-seq 2 4] [--per-video 1 2] [--mot qd byte none] [--steps 20]

The batch workload: n_seq videos (make_video seeds 0..n_seq-1), each with `per_video` targets (one per object, added on frame 0) and
the MOT arm, three sides in the same process, all pipelined (submit(t + 1) before collect(t), the association included):
UnicornUnifiedBatch over all videos; n_seq UnicornUnifiedTrackers stepped in turn; UnicornSOTBatch over all targets (each fed its
video's frame) plus UnicornMOTBatch(n_seq) (the SOT batch of step t is collected before its next submit).  The device-only step is
the graph replays of every side's drivers with their input copies.  Besides the ms per step, each side reports the aggregate
video-frames/s (n_seq / step time).  One JSON line per (config, n_seq, per_video, mot).

    python tools/bench_unified.py --workload mask-batch [--configs ...] [--n-seq 2 4] [--objects 1 3] [--mots on off] [--steps 20]

The mask-batch workload: n_seq videos of mixed original sizes (1080x1920 and 480x640 in turn, make_video seeds 0..n_seq-1, each
letterboxed once on the host to 800x1280 uint8 and kept on the device), each with `objects` VOS objects (added on frame 0, in one
group) and optionally the MOTS arm, on unicorn_track_large_mask and unicorn_track_large_mot_challenge_mask.  Three sides in the same
process: UnicornUnifiedMaskBatch over all videos and n_seq UnicornUnifiedMaskTrackers stepped in turn, both pipelined (submit(t + 1)
before collect(t)); UnicornVOSBatch (synchronous per step) plus UnicornMOTSBatch (pipelined).  A step includes the VOS result assembly
of every video, the MOTS association and the mask encode.  The device-only step is every side's graph replays with their input
copies plus the result assemblies outside the graphs.  Launches per step count the kernels of the graphs plus the launches outside
them.  One JSON line per (config, n_seq, objects, mots)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import types

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=["box", "mask", "batch", "mask-batch"], default="box")
    ap.add_argument("--configs", nargs="+", default=None)
    ap.add_argument("--size", type=int, nargs=2, default=(800, 1280))
    ap.add_argument("--targets", type=int, nargs="+", default=[1, 2, 4])
    ap.add_argument("--mot", nargs="+", default=["qd", "byte", "none"], choices=["qd", "byte", "none"])
    ap.add_argument("--objects", type=int, nargs="+", default=[1, 3])
    ap.add_argument("--mots", nargs="+", default=["on", "off"], choices=["on", "off"])
    ap.add_argument("--orig", type=int, nargs=2, default=(1080, 1920))
    ap.add_argument("--n-seq", type=int, nargs="+", default=[2, 4])
    ap.add_argument("--per-video", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": torch.cuda.get_device_name(), "nvidia_smi": q}), flush=True)
    if args.workload in ("mask", "mask-batch"):
        args.configs = args.configs or ["unicorn_track_large_mask", "unicorn_track_large_mot_challenge_mask"]
        return mask(args) if args.workload == "mask" else mask_batch(args)
    args.configs = args.configs or ["unicorn_track_large", "unicorn_track_r50"]
    if args.workload == "batch":
        return batch(args)
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.mot import UnicornMOTTracker
    from unicorn_b200.sot import UnicornSOTBatch
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    from unicorn_b200.tracker.byte_tracker import BYTETracker
    from unicorn_b200.unified import UnicornUnifiedTracker
    from unicorn_b200.weights import make_state_dict

    H, W = args.size
    bargs = types.SimpleNamespace(track_thresh=0.5, track_buffer=30, match_thresh=0.8, mot20=False)
    new_tracker = {"qd": lambda: QuasiDenseEmbedTracker(), "byte": lambda: BYTETracker(bargs), None: lambda: None}
    to_u8 = lambda f: f.round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()  # noqa: E731
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for cfg in args.configs:
        eng = UnicornEngine(make_state_dict(cfg, 0), cfg)
        frames, boxes = make_video(5, H, W, seed=0, n_obj=6)
        ref = to_u8(frames[0:1]).cuda()
        steps_u8 = [to_u8(frames[1 + t:2 + t]).cuda() for t in range(4)]  # [1,H,W,3]
        for K in args.targets:
            copies = [f.expand(K, -1, -1, -1).contiguous() for f in steps_u8]
            for mot in [None if m == "none" else m for m in args.mot]:
                sides = {}
                # ---- one backbone pass per frame
                m0 = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                un = UnicornUnifiedTracker(eng, (H, W), K, mot=mot, tracker=new_tracker[mot]())
                for k in range(K):
                    un.add_target(k, boxes[0, k])
                un.step_tensor(ref)

                def un_round(steps, un=un):
                    un.submit(steps_u8[0])
                    for t in range(steps):
                        if t + 1 < steps:
                            un.submit(steps_u8[(t + 1) % 4])
                        un.collect((H, W))

                def un_replay(t, un=un):
                    un._slot.img_in_u8.copy_(steps_u8[t % 4], non_blocking=True)
                    un._slot.graph.replay()
                un_round(4)
                sides["unified"] = (un_round, un_replay, un.launches_per_frame, torch.cuda.max_memory_allocated() - m0)
                # ---- today's drivers, each with its own backbone pass
                m0 = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                sb = UnicornSOTBatch(eng, (H, W), K)
                for k in range(K):
                    sb.initialize_tensor(k, ref, boxes[0, k])
                mt = UnicornMOTTracker(eng, (H, W), assoc=mot, tracker=new_tracker[mot](), use_graph=True) if mot else None

                def two_round(steps, sb=sb, mt=mt):
                    if mt:
                        mt.submit(steps_u8[0])
                    for t in range(steps):
                        sb.submit(copies[t % 4])
                        if mt and t + 1 < steps:
                            mt.submit(steps_u8[(t + 1) % 4])
                        sb.collect()
                        if mt:
                            mt.collect((H, W))

                def two_replay(t, sb=sb, mt=mt):
                    sb.slot.img_in_u8.copy_(copies[t % 4], non_blocking=True)
                    sb.slot.graph.replay()
                    if mt:
                        c = mt._ctxs[t % 2]
                        c.img_in_u8.copy_(steps_u8[t % 4], non_blocking=True)
                        c.graph.replay()
                two_round(4)
                launches = sb.launches_per_frame + (mt._b.launches_per_frame if mt else 0)
                sides["two_drivers"] = (two_round, two_replay, launches, torch.cuda.max_memory_allocated() - m0)
                line = {"config": cfg, "size": [H, W], "targets": K, "mot": mot or "none"}
                line.update(compare(sides, args, e0, e1))
                print(json.dumps(line), flush=True)
                del sides, un, sb, mt, un_round, un_replay, two_round, two_replay
                torch.cuda.empty_cache()
        del eng
        torch.cuda.empty_cache()


def compare(sides, args, e0, e1):
    """Times every side of `sides` {name: (round(steps), replay(t), launches, added bytes)}: rounds alternate between the sides."""
    times = {key: [] for key in sides}
    for _ in range(args.rounds):
        for key, (run, *_rest) in sides.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(args.steps)
            torch.cuda.synchronize()
            times[key].append(time.perf_counter() - t0)
    line = {}
    for key, (_, replay, launches, mem) in sides.items():
        torch.cuda.synchronize()
        e0.record()
        for t in range(args.steps):
            replay(t)
        e1.record()
        torch.cuda.synchronize()
        ms = [1e3 * t / args.steps for t in times[key]]
        line[key] = {"ms_per_step": round(statistics.median(ms), 2), "ms_per_step_min_max": [round(min(ms), 2), round(max(ms), 2)],
                     "device_ms_per_step": round(e0.elapsed_time(e1) / args.steps, 2), "launches_per_step": launches,
                     "added_peak_alloc_gib": round(mem / 2 ** 30, 2)}
    first, *others = sides
    for key in others:  # each other side's step time over the first side's
        line[f"{key}_over_{first}"] = round(line[key]["ms_per_step"] / line[first]["ms_per_step"], 3)
    line.update(steps=args.steps, rounds=args.rounds)
    return line


def mask(args):
    from unicorn_b200 import _lib, shared_ops
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.mots import UnicornMOTSTracker
    from unicorn_b200.sot import preprocess
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.unified import UnicornUnifiedMaskTracker
    from unicorn_b200.vos import UnicornVOSTrack
    from unicorn_b200.weights import make_state_dict

    H, W = args.size
    h0, w0 = args.orig
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    frames, boxes = make_video(5, h0, w0, seed=0, n_obj=6)
    rgb = [f.permute(1, 2, 0).flip(-1).round().clamp(0, 255).to(torch.uint8).numpy().copy() for f in frames]
    lb = [preprocess(im, (H, W)) for im in rgb]
    r = lb[0][1]
    ref = lb[0][0].cuda()
    steps_u8 = [f.cuda() for f, _ in lb[1:]]  # [1,H,W,3] letterboxed, resident on the device

    def outside(step, n=4):
        """Launches per step outside the graphs (result assembly, encode), counted over n steps."""
        l0 = _lib.LAUNCHES
        for t in range(n):
            step(t)
        return (_lib.LAUNCHES - l0) / n

    for cfg in args.configs:
        eng = UnicornEngine(make_state_dict(cfg, 0), cfg)
        for K in args.objects:
            objs = {k + 1: boxes[0, k] * r for k in range(K)}
            for mots in [m == "on" for m in args.mots]:
                sides = {}
                # ---- one backbone pass per frame
                m0 = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                un = UnicornUnifiedMaskTracker(eng, (H, W), (h0, w0), K, 1, mots=mots)
                un.add_objects(objs)
                un.step_tensor(ref)

                def un_round(steps, un=un):
                    un.submit(steps_u8[0])
                    for t in range(steps):
                        if t + 1 < steps:
                            un.submit(steps_u8[(t + 1) % 4])
                        un.collect()

                def un_replay(t, un=un):
                    s = un._ring.slots[t % 2]
                    s.img_in_u8.copy_(steps_u8[t % 4], non_blocking=True)
                    s.graph.replay()
                    shared_ops.vos_aggregate_batched([([s.vos_masks[k] for _, k in s.objs[0]], None, [o for o, _ in s.objs[0]], un.r, s.soft[0],
                                                       s.seg[0])], H, W)
                un_round(4)
                launches = un.launches_per_frame + outside(lambda t: un.step_tensor(steps_u8[t % 4]))
                sides["unified"] = (un_round, un_replay, launches, torch.cuda.max_memory_allocated() - m0)
                # ---- today's drivers, each with its own backbone and mask-branch pass
                m0 = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                vt = UnicornVOSTrack(eng, (H, W), use_graph=True, depth=2)
                vt.initialize_tensor(ref, objs, orig_size=(h0, w0), r=r)
                mt = UnicornMOTSTracker(eng, (H, W), use_graph=True) if mots else None
                mots_launches = 0
                if mt:  # the first MOTS step runs eagerly: its launches are those its graphs replay
                    l0 = _lib.LAUNCHES
                    mt.submit(ref, h0, w0)
                    mots_launches = _lib.LAUNCHES - l0
                    mt.collect()

                def two_round(steps, vt=vt, mt=mt):
                    vt.submit(steps_u8[0])
                    if mt:
                        mt.submit(steps_u8[0], h0, w0)
                    for t in range(steps):
                        if t + 1 < steps:
                            vt.submit(steps_u8[(t + 1) % 4])
                            if mt:
                                mt.submit(steps_u8[(t + 1) % 4], h0, w0)
                        vt.collect()
                        if mt:
                            mt.collect()

                def two_replay(t, vt=vt, mt=mt):
                    s = vt._workers[t % 2]
                    s.img_in_u8.copy_(steps_u8[t % 4], non_blocking=True)
                    s.graph.replay()
                    if mt:
                        c = mt._ctxs[t % 2]
                        c.img_in_u8.copy_(steps_u8[t % 4], non_blocking=True)
                        c.graph.replay()
                two_round(6)

                def two_step(t, vt=vt, mt=mt):
                    vt.submit(steps_u8[t % 4])
                    vt.collect()
                    if mt:
                        mt.step_tensor(steps_u8[t % 4], h0, w0)
                launches = vt.launches_per_frame + mots_launches + outside(two_step)
                sides["two_drivers"] = (two_round, two_replay, launches, torch.cuda.max_memory_allocated() - m0)
                line = {"config": cfg, "size": [H, W], "orig": [h0, w0], "objects": K, "mots": mots}
                line.update(compare(sides, args, e0, e1))
                print(json.dumps(line), flush=True)
                del sides, un, vt, mt, un_round, un_replay, two_round, two_replay, two_step
                torch.cuda.empty_cache()
        del eng
        torch.cuda.empty_cache()


def batch(args):
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.mot import UnicornMOTBatch
    from unicorn_b200.sot import UnicornSOTBatch
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.tracker import QuasiDenseEmbedTracker
    from unicorn_b200.tracker.byte_tracker import BYTETracker
    from unicorn_b200.unified import UnicornUnifiedBatch, UnicornUnifiedTracker
    from unicorn_b200.weights import make_state_dict

    H, W = args.size
    bargs = types.SimpleNamespace(track_thresh=0.5, track_buffer=30, match_thresh=0.8, mot20=False)
    new_tracker = {"qd": lambda: QuasiDenseEmbedTracker(), "byte": lambda: BYTETracker(bargs), None: lambda: None}
    to_u8 = lambda f: f.round().clamp(0, 255).to(torch.uint8).permute(0, 2, 3, 1).contiguous()  # noqa: E731
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    vids = [make_video(5, H, W, seed=i, n_obj=6) for i in range(max(args.n_seq))]
    refs_all = [to_u8(f[0:1]).cuda() for f, _ in vids]  # [1,H,W,3] per video
    steps_all = [[to_u8(f[1 + t:2 + t]).cuda() for t in range(4)] for f, _ in vids]
    for cfg in args.configs:
        eng = UnicornEngine(make_state_dict(cfg, 0), cfg)
        for n in args.n_seq:
            refs, steps = refs_all[:n], steps_all[:n]
            ref_b = torch.cat(refs)
            steps_b = [torch.cat([steps[i][t] for i in range(n)]) for t in range(4)]  # [n,H,W,3]
            for T in args.per_video:
                targets = [(i, k) for i in range(n) for k in range(T)]  # (video, object) per target
                copies = [torch.cat([steps[i][t] for i, _ in targets]) for t in range(4)]  # one frame copy per target
                for mot in [None if m == "none" else m for m in args.mot]:
                    sides = {}
                    # ---- one step for every video: UnicornUnifiedBatch
                    m0 = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    ub = UnicornUnifiedBatch(eng, (H, W), n, n * T, mot=mot)
                    for i in range(n):
                        ub.start(i, new_tracker[mot]())
                    for i, k in targets:
                        ub.add_target(i, k, vids[i][1][0, k])
                    ub.step_tensor(ref_b)

                    def ub_round(nsteps, ub=ub):
                        ub.submit(steps_b[0])
                        for t in range(nsteps):
                            if t + 1 < nsteps:
                                ub.submit(steps_b[(t + 1) % 4])
                            ub.collect([(H, W)] * n)

                    def ub_replay(t, ub=ub):
                        ub._slot.img_in_u8.copy_(steps_b[t % 4], non_blocking=True)
                        ub._slot.graph.replay()
                    ub_round(4)
                    sides["batch"] = (ub_round, ub_replay, ub.launches_per_frame, torch.cuda.max_memory_allocated() - m0)
                    # ---- one UnicornUnifiedTracker per video, stepped in turn
                    m0 = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    uts = []
                    for i in range(n):
                        ut = UnicornUnifiedTracker(eng, (H, W), T, mot=mot, tracker=new_tracker[mot]())
                        for k in range(T):
                            ut.add_target(k, vids[i][1][0, k])
                        ut.step_tensor(refs[i])
                        uts.append(ut)

                    def ut_round(nsteps, uts=uts):
                        for i, ut in enumerate(uts):
                            ut.submit(steps[i][0])
                        for t in range(nsteps):
                            for i, ut in enumerate(uts):
                                if t + 1 < nsteps:
                                    ut.submit(steps[i][(t + 1) % 4])
                                ut.collect((H, W))

                    def ut_replay(t, uts=uts):
                        for i, ut in enumerate(uts):
                            ut._slot.img_in_u8.copy_(steps[i][t % 4], non_blocking=True)
                            ut._slot.graph.replay()
                    ut_round(4)
                    sides["trackers"] = (ut_round, ut_replay, sum(ut.launches_per_frame for ut in uts),
                                         torch.cuda.max_memory_allocated() - m0)
                    # ---- UnicornSOTBatch over all targets plus UnicornMOTBatch over the videos
                    m0 = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    sb = UnicornSOTBatch(eng, (H, W), len(targets))
                    for j, (i, k) in enumerate(targets):
                        sb.initialize_tensor(j, refs[i], vids[i][1][0, k])
                    mt = None
                    if mot:
                        mt = UnicornMOTBatch(eng, (H, W), n, assoc=mot, use_graph=True)
                        for i in range(n):
                            mt.start(i, new_tracker[mot]())
                        mt.step_tensor(ref_b)

                    def sm_round(nsteps, sb=sb, mt=mt):
                        if mt:
                            mt.submit(steps_b[0])
                        for t in range(nsteps):
                            sb.submit(copies[t % 4])
                            if mt and t + 1 < nsteps:
                                mt.submit(steps_b[(t + 1) % 4])
                            sb.collect()
                            if mt:
                                mt.collect([(H, W)] * n)

                    def sm_replay(t, sb=sb, mt=mt):
                        sb.slot.img_in_u8.copy_(copies[t % 4], non_blocking=True)
                        sb.slot.graph.replay()
                        if mt:
                            c = mt._ctxs[t % 2]
                            c.img_in_u8.copy_(steps_b[t % 4], non_blocking=True)
                            c.graph.replay()
                    sm_round(4)
                    launches = sb.launches_per_frame + (mt.launches_per_frame if mt else 0)
                    sides["sot_mot"] = (sm_round, sm_replay, launches, torch.cuda.max_memory_allocated() - m0)
                    line = {"config": cfg, "size": [H, W], "n_seq": n, "per_video": T, "mot": mot or "none"}
                    line.update(compare(sides, args, e0, e1))
                    for key in sides:
                        line[key]["video_frames_per_s"] = round(1e3 * n / line[key]["ms_per_step"], 1)
                    print(json.dumps(line), flush=True)
                    del sides, ub, uts, sb, mt, ub_round, ub_replay, ut_round, ut_replay, sm_round, sm_replay
                    torch.cuda.empty_cache()
        del eng
        torch.cuda.empty_cache()


def mask_batch(args):
    from unicorn_b200 import _lib, ops, shared_ops
    from unicorn_b200.engine import UnicornEngine
    from unicorn_b200.mots import UnicornMOTSBatch
    from unicorn_b200.sot import preprocess
    from unicorn_b200.synthetic import make_video
    from unicorn_b200.unified import UnicornUnifiedMaskBatch, UnicornUnifiedMaskTracker
    from unicorn_b200.vos import UnicornVOSBatch
    from unicorn_b200.weights import make_state_dict

    H, W = args.size
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    origs = [(1080, 1920), (480, 640)]
    vids = []  # per video: (original size, r, letterboxed reference [1,H,W,3], 4 letterboxed steps, frame-0 boxes in resized coordinates)
    for i in range(max(args.n_seq)):
        h0, w0 = origs[i % 2]
        frames, boxes = make_video(5, h0, w0, seed=i, n_obj=6)
        rgb = [f.permute(1, 2, 0).flip(-1).round().clamp(0, 255).to(torch.uint8).numpy().copy() for f in frames]
        lb = [preprocess(im, (H, W)) for im in rgb]
        r = lb[0][1]
        vids.append(((h0, w0), r, lb[0][0].cuda(), [f.cuda() for f, _ in lb[1:]], boxes[0] * r))

    def outside(step, n=4):
        """Launches per step outside the graphs (result assembly, encode), counted over n steps."""
        l0 = _lib.LAUNCHES
        for t in range(n):
            step(t)
        return (_lib.LAUNCHES - l0) / n

    for cfg in args.configs:
        eng = UnicornEngine(make_state_dict(cfg, 0), cfg)
        for n in args.n_seq:
            vs = vids[:n]
            ref_b = torch.cat([v[2] for v in vs])
            steps_b = [torch.cat([v[3][t] for v in vs]) for t in range(4)]  # [n,H,W,3]
            sizes = [v[0] for v in vs]
            for K in args.objects:
                objs = [{k + 1: v[4][k] for k in range(K)} for v in vs]
                for mots in [m == "on" for m in args.mots]:
                    sides = {}
                    # ---- one step for every video: UnicornUnifiedMaskBatch
                    m0 = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    ub = UnicornUnifiedMaskBatch(eng, (H, W), n, n * K, n, mots=mots)
                    for i, v in enumerate(vs):
                        ub.start(i, v[0])
                        ub.add_objects(i, objs[i])
                    ub.step_tensor(ref_b)

                    def ub_round(nsteps, ub=ub):
                        ub.submit(steps_b[0])
                        for t in range(nsteps):
                            if t + 1 < nsteps:
                                ub.submit(steps_b[(t + 1) % 4])
                            ub.collect()

                    def ub_replay(t, ub=ub):
                        s = ub._ring.slots[t % 2]
                        s.img_in_u8.copy_(steps_b[t % 4], non_blocking=True)
                        s.graph.replay()
                        shared_ops.vos_aggregate_batched([([s.vos_masks[k] for _, k in s.objs[i]], None, [o for o, _ in s.objs[i]], s.r[i], s.soft[i],
                                                    s.seg[i]) for i in range(n)], H, W)
                    ub_round(4)
                    launches = ub.launches_per_frame + outside(lambda t, ub=ub: ub.step_tensor(steps_b[t % 4]))
                    sides["batch"] = (ub_round, ub_replay, launches, torch.cuda.max_memory_allocated() - m0)
                    # ---- one UnicornUnifiedMaskTracker per video, stepped in turn
                    m0 = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    uts = []
                    for i, v in enumerate(vs):
                        ut = UnicornUnifiedMaskTracker(eng, (H, W), v[0], K, 1, mots=mots)
                        ut.add_objects(objs[i])
                        ut.step_tensor(v[2])
                        uts.append(ut)

                    def ut_round(nsteps, uts=uts):
                        for i, ut in enumerate(uts):
                            ut.submit(vs[i][3][0])
                        for t in range(nsteps):
                            for i, ut in enumerate(uts):
                                if t + 1 < nsteps:
                                    ut.submit(vs[i][3][(t + 1) % 4])
                                ut.collect()

                    def ut_replay(t, uts=uts):
                        for i, ut in enumerate(uts):
                            s = ut._ring.slots[t % 2]
                            s.img_in_u8.copy_(vs[i][3][t % 4], non_blocking=True)
                            s.graph.replay()
                            shared_ops.vos_aggregate_batched([([s.vos_masks[k] for _, k in s.objs[0]], None, [o for o, _ in s.objs[0]], ut.r,
                                                               s.soft[0], s.seg[0])], H, W)
                    ut_round(4)

                    def ut_step(t, uts=uts):
                        for i, ut in enumerate(uts):
                            ut.step_tensor(vs[i][3][t % 4])
                    launches = sum(ut.launches_per_frame for ut in uts) + outside(ut_step)
                    sides["trackers"] = (ut_round, ut_replay, launches, torch.cuda.max_memory_allocated() - m0)
                    # ---- UnicornVOSBatch over the videos plus UnicornMOTSBatch over the videos
                    m0 = torch.cuda.memory_allocated()
                    torch.cuda.reset_peak_memory_stats()
                    vb = UnicornVOSBatch(eng, (H, W), n, n * K, n)
                    for i, v in enumerate(vs):
                        vb.initialize_tensor(i, v[2], objs[i], orig_size=v[0], r=v[1])
                    vb.track_tensor(steps_b[0])  # captures the graph
                    mb, mots_launches = None, 0
                    if mots:
                        mb = UnicornMOTSBatch(eng, (H, W), n, use_graph=True)
                        for i in range(n):
                            mb.start(i)
                        mb.step_tensor(ref_b, sizes)  # the first step runs eagerly: its launches are those its graphs replay
                        mots_launches = mb.launches_per_frame

                    def vm_round(nsteps, vb=vb, mb=mb):
                        if mb:
                            mb.submit(steps_b[0], sizes)
                        for t in range(nsteps):
                            vb.track_tensor(steps_b[t % 4])
                            if mb and t + 1 < nsteps:
                                mb.submit(steps_b[(t + 1) % 4], sizes)
                            if mb:
                                mb.collect()

                    def vm_replay(t, vb=vb, mb=mb):
                        vb.slot.img_in_u8.copy_(steps_b[t % 4], non_blocking=True)
                        vb.slot.graph.replay()
                        for sq in vb.seqs:
                            ids = sq.obj_ids
                            ops.vos_aggregate([vb.masks[sq.obj_slot[o]] for o in ids], None, ids, H, W, sq.r, sq.soft, sq.seg)
                        if mb:
                            c = mb._ctxs[t % 2]
                            c.img_in_u8.copy_(steps_b[t % 4], non_blocking=True)
                            c.graph.replay()
                    vm_round(4)

                    def vm_step(t, vb=vb, mb=mb):
                        vb.track_tensor(steps_b[t % 4])
                        if mb:
                            mb.step_tensor(steps_b[t % 4], sizes)
                    launches = vb.launches_per_frame + mots_launches + outside(vm_step)
                    sides["vos_mots"] = (vm_round, vm_replay, launches, torch.cuda.max_memory_allocated() - m0)
                    line = {"config": cfg, "size": [H, W], "origs": sizes, "n_seq": n, "objects": K, "mots": mots}
                    line.update(compare(sides, args, e0, e1))
                    for key in sides:
                        line[key]["video_frames_per_s"] = round(1e3 * n / line[key]["ms_per_step"], 1)
                    print(json.dumps(line), flush=True)
                    del sides, ub, uts, vb, mb, ub_round, ub_replay, ut_round, ut_replay, ut_step, vm_round, vm_replay, vm_step
                    torch.cuda.empty_cache()
        del eng
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
