"""Frames/s of the other BASELINE.json workloads on ONE H100 (bench.py measures configs[1]):
  mot : configs[2] — ConvNeXt-L MOT detector + embedding path at 1536x2048 (mode="whole", NMS, embedding sampling), then
        (a) the QDTrack association of the reference's MOT evaluator on the model's own detections and
        (b) ByteTrack association on 100 synthetic objects per frame (random weights give few detections of their own).
  vos : configs[3] — ConvNeXt-L + CondInst mask head at 800x1280, n objects propagated from the first frame.
Eager launches (no CUDA graph: the association step returns to the host every frame), wall clock around synchronised
steps, synthetic video, seeded weights.
  r50 : the SOT frame at 800x1280 of unicorn_track_r50 and, in the same process for comparison, of unicorn_track_large: CUDA graphs,
        one frame and three frames in flight, three alternating rounds.
  mots: the MOTS frame of unicorn_track_large_mot_challenge_mask at 800x1280 from 1080x1920 originals, sequential eager and pipelined
        with CUDA graphs, the host half it replaced on the same masks, and the mask encoding alone on 20 and 50 synthetic instances
        (uc_mots_encode against results.mots_frame_result).
usage: bench_workloads.py mot|vos|r50|mots [frames]"""
import json, os, sys, time, types
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from unicorn_b200 import _lib
from unicorn_b200.engine import UnicornEngine
from unicorn_b200.synthetic import make_video, make_detections
from unicorn_b200.weights import make_state_dict

what = sys.argv[1] if len(sys.argv) > 1 else "mot"
n = int(sys.argv[2]) if len(sys.argv) > 2 else 12
dev = "cuda"


def timed(fn, n, warm=3):
    for i in range(warm):
        fn(i)
    torch.cuda.synchronize()
    l0, t0 = _lib.LAUNCHES, time.perf_counter()
    for i in range(n):
        fn(warm + i)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return n / dt, 1e3 * dt / n, (_lib.LAUNCHES - l0) // n


if what == "mot":
    from unicorn_b200.mot import UnicornMOTTracker
    from unicorn_b200.tracker.byte_tracker import BYTETracker
    H, W = 1536, 2048
    cfg = "unicorn_track_large_mot_challenge"
    eng = UnicornEngine(make_state_dict(cfg, 0), cfg)
    frames, _ = make_video(4, H, W, seed=0, n_obj=6)
    frames = [f[None].to(dev) for f in frames]
    args = types.SimpleNamespace(track_thresh=0.5, track_buffer=30, match_thresh=0.8, mot20=False)
    dets100 = make_detections(n_frames=n + 8, n_obj=100, seed=3, W=float(W), H=float(H))

    def pipelined(trk, extra=None):
        """submit(t+1); collect(t): host association of frame t overlaps the device work of frame t+1"""
        trk.submit(frames[0])
        def step(i):
            trk.submit(frames[(i + 1) % 4])
            trk.collect()
            if extra:
                extra(i)
        r = timed(step, n, warm=5)
        trk.collect()
        return r

    trk = UnicornMOTTracker(eng, (H, W))
    fps, ms, launches = timed(lambda i: trk.step_tensor(frames[i % 4]), n)
    print(json.dumps({"workload": "configs[2] MOT 1536x2048 ConvNeXt-L: detector + embedding + QDTrack association, sequential eager",
                      "frames_per_s": round(fps, 2), "ms_per_frame": round(ms, 2), "kernels_per_frame": launches, "n_gpus": 1}))
    trk = UnicornMOTTracker(eng, (H, W), use_graph=True)
    fps, ms, launches = pipelined(trk)
    print(json.dumps({"workload": "configs[2] same, device half as CUDA graphs, association of frame t overlapped with frame t+1",
                      "frames_per_s": round(fps, 2), "ms_per_frame": round(ms, 2), "kernels_per_frame": launches, "n_gpus": 1}))
    # ByteTrack arm: detector (no embedding branch) + BYTETracker.update.  Seeded random weights give only a handful of
    # detections, so a second tracker is fed 100 synthetic objects per frame inside the same loop: the measured rate
    # includes the host cost of a 100-object association while the device runs the next frame.
    bt100 = BYTETracker(args, device=dev)
    trk = UnicornMOTTracker(eng, (H, W), assoc="byte", tracker=BYTETracker(args, device=dev), use_graph=True)
    fps, ms, launches = pipelined(trk, extra=lambda i: bt100.update(dets100[i][0].numpy(), (H, W), (H, W)))
    print(json.dumps({"workload": "configs[2] MOT 1536x2048 ConvNeXt-L detector (CUDA graphs) + ByteTrack association of 100 synthetic "
                                  "objects per frame, pipelined", "frames_per_s": round(fps, 2), "ms_per_frame": round(ms, 2),
                      "kernels_per_frame": launches, "n_gpus": 1}))
    bt = BYTETracker(args, device=dev)
    fps2, ms2, l2 = timed(lambda i: bt.update(dets100[i][0].numpy(), (H, W), (H, W)), n)
    print(json.dumps({"workload": "configs[2] ByteTrack update alone, 100 synthetic objects per frame (host Kalman + LAP, IoU on the GPU)",
                      "frames_per_s": round(fps2, 1), "ms_per_frame": round(ms2, 3), "kernels_per_frame": l2}))
elif what == "r50":
    import subprocess
    from unicorn_b200.sot import UnicornSOTTrack
    H, W = 800, 1280
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": torch.cuda.get_device_name(), "nvidia_smi": q}))
    frames, boxes = make_video(4, H, W, seed=0)
    frames = [f[None].pin_memory() for f in frames]
    trackers = {}
    for cfg in ("unicorn_track_r50", "unicorn_track_large"):
        eng = UnicornEngine(make_state_dict(cfg, 0), cfg)
        for depth in (1, 3):
            trk = UnicornSOTTrack(eng, (H, W), depth=depth)
            trk.initialize_tensor(frames[0], boxes[0, 0])
            trackers[cfg, depth] = trk

    def in_flight(trk):
        def step(i):
            if trk.depth == 1:
                trk.track_tensor(frames[1 + i % 3])
                return
            if trk._ring.submitted - trk._ring.collected == trk.depth:
                trk.collect()
            trk.submit(frames[1 + i % 3])
        return step

    for rnd in range(3):
        for (cfg, depth), trk in trackers.items():
            fps, ms, launches = timed(in_flight(trk), n, warm=6)
            while trk._ring.collected < trk._ring.submitted:
                trk.collect()
            print(json.dumps({"workload": f"SOT 800x1280 {cfg}, CUDA graphs, {depth} frame(s) in flight", "round": rnd,
                              "frames_per_s": round(fps, 2), "ms_per_frame": round(ms, 2), "kernels_per_frame": launches, "n_gpus": 1}))
elif what == "mots":
    import subprocess
    import torch.nn.functional as F
    from unicorn_b200 import results as R
    from unicorn_b200.mots import MaskEncoder, UnicornMOTSTracker
    H, W, h0, w0 = 800, 1280, 1080, 1920
    scale = min(H / float(h0), W / float(w0))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"card": torch.cuda.get_device_name(), "nvidia_smi": q}))
    cfg = "unicorn_track_large_mot_challenge_mask"
    eng = UnicornEngine(make_state_dict(cfg, 0), cfg)
    frames, _ = make_video(4, H, W, seed=1, n_obj=6)
    frames = [f[None].to(dev) for f in frames]
    trk = UnicornMOTSTracker(eng, (H, W))
    tracked = []
    fps, ms, launches = timed(lambda i: tracked.append(len(trk.step_tensor(frames[i % 4], h0, w0)[1])), n)
    print(json.dumps({"workload": f"MOTS 800x1280 {cfg} from 1080x1920 frames: detector + masks + QDTrack + device RLE, sequential eager",
                      "frames_per_s": round(fps, 2), "ms_per_frame": round(ms, 2), "kernels_per_frame": launches,
                      "tracks_per_frame": tracked[-n:], "n_gpus": 1}))

    def host_half(i):
        """the host half this driver replaced, on the driver's own masks: resize at the original size, read back, overlap, RLE"""
        last = trk.last
        m = torch.zeros(0, h0, w0, dtype=torch.bool)
        if last["rows"].numel():
            m = F.interpolate(last["masks"][last["rows"]][:, None], scale_factor=1 / scale, mode="bilinear",
                              align_corners=False)[:, 0, :h0, :w0] > trk.mask_thres
        R.mots_frame_result(i, last["boxes"], last["ids"], m.cpu(), h0, w0, trk.min_box_area)
    trk.step_tensor(frames[0], h0, w0)
    fps, ms, _ = timed(host_half, n)
    print(json.dumps({"workload": "MOTS old host half on the same frame's masks (F.interpolate + .cpu() + results.mots_frame_result)",
                      "tracks": int(trk.last["rows"].numel()), "ms_per_frame": round(ms, 3)}))
    trk = UnicornMOTSTracker(eng, (H, W), use_graph=True)
    trk.submit(frames[0], h0, w0)

    def step(i):
        trk.submit(frames[(i + 1) % 4], h0, w0)
        trk.collect()
    fps, ms, launches = timed(step, n, warm=5)
    trk.collect()
    print(json.dumps({"workload": "MOTS same, device half as CUDA graphs, host half of frame t overlapped with frame t+1",
                      "frames_per_s": round(fps, 2), "ms_per_frame": round(ms, 2), "kernels_per_frame": launches, "n_gpus": 1}))
    # seeded weights give few detections: the encode alone on synthetic elliptical instances at the original 1080x1920
    yy, xx = torch.meshgrid(torch.arange(H, device=dev, dtype=torch.float32), torch.arange(W, device=dev, dtype=torch.float32), indexing="ij")
    g = torch.Generator().manual_seed(0)
    for k in (20, 50):
        p = torch.rand(k, 4, generator=g).tolist()
        masks = torch.stack([(((yy - a * H) / (40 + b * H / 4)) ** 2 + ((xx - c * W) / (40 + d * W / 4)) ** 2 < 1).float()
                             for a, b, c, d in p]).contiguous()
        boxes = torch.tensor([[0.0, 0.0, 100.0, 100.0, 1.0]] * k)
        ids = torch.arange(k)
        enc = MaskEncoder(k, dev)
        dev_ms = timed(lambda i: enc(masks, list(range(k)), [True] * k, 0.3, scale, h0, w0), 2 * n)[1]
        got = enc(masks, list(range(k)), [True] * k, 0.3, scale, h0, w0)

        def host(i):
            m = F.interpolate(masks[:, None], scale_factor=1 / scale, mode="bilinear", align_corners=False)[:, 0, :h0, :w0] > 0.3
            return R.mots_frame_result(i, boxes, ids, m.cpu(), h0, w0, 0)
        host_ms = timed(host, 3, warm=1)[1]
        same = host(0)[5] == got
        print(json.dumps({"workload": f"MOTS encode alone, {k} instances, 1080x1920", "uc_mots_encode_ms": round(dev_ms, 3),
                          "host_mots_frame_result_ms": round(host_ms, 1), "identical_strings": same}))
else:
    from unicorn_b200.vos import UnicornVOSTrack
    H, W = 800, 1280
    cfg = "unicorn_track_large_mask"
    eng = UnicornEngine(make_state_dict(cfg, 0), cfg)
    for n_obj in (1, 3):
        frames, boxes = make_video(4, H, W, seed=1, n_obj=n_obj)
        frames = [f[None].to(dev) for f in frames]
        trk = UnicornVOSTrack(eng, (H, W))
        trk.initialize_tensor(frames[0], {o + 1: boxes[0, o].tolist() for o in range(n_obj)})
        fps, ms, launches = timed(lambda i: trk.track_tensor(frames[1 + i % 3]), n)
        print(json.dumps({"workload": f"configs[3] VOS 800x1280 ConvNeXt-L + CondInst mask head, {n_obj} object(s) (eager)",
                          "frames_per_s": round(fps, 2), "ms_per_frame": round(ms, 2), "kernels_per_frame": launches, "n_gpus": 1}))
