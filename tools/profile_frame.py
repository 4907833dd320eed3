"""Run init + N eager (non-graph) SOT frames of a config, then print where the device time of one more frame goes: per-kernel
device time from torch.profiler (CUDA activities), grouped by kernel name, largest first; their sum next to the step time of the
same frame replayed as a CUDA graph; and the per-layer table of the convolutions (block_n code, launches, device time).

usage: profile_frame.py [--no-pdl] [config] [frames] [tuning table to save]

--no-pdl sets UC_PDL=0 before the library is loaded.  With programmatic dependent launch on, a kernel's CTAs may become resident
while its predecessor drains and wait there, and the profiler counts that wait as the kernel's duration; with it off, kernels
run in plain stream order and each duration is the kernel's own.  UC_CONV_TRACE=FILE also writes the conv trace as JSON."""
import os, re, sys
args = [a for a in sys.argv[1:] if a != "--no-pdl"]
if "--no-pdl" in sys.argv:
    os.environ["UC_PDL"] = "0"
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from unicorn_b200 import _lib, ops
from unicorn_b200.engine import UnicornEngine
from unicorn_b200.sot import UnicornSOTTrack
from unicorn_b200.synthetic import make_video
from unicorn_b200.weights import make_state_dict
name = args[0] if len(args) > 0 else "unicorn_track_large"
nfr = int(args[1]) if len(args) > 1 else 2
H, W = (320, 320) if "tiny" in name else (800, 1280)
sd = make_state_dict(name, 0)
frames, boxes = make_video(nfr + 1, H, W, seed=0)
eng = UnicornEngine(sd, name)
trk = UnicornSOTTrack(eng, (H, W), use_graph=False)
trk.initialize_tensor(frames[0:1], boxes[0, 0])
print("launches after init", _lib.LAUNCHES, "PDL", "off" if os.environ.get("UC_PDL", "1")[:1] == "0" else "on")
for i in range(nfr):
    l0 = _lib.LAUNCHES
    trk.track_tensor(frames[1 + i:2 + i])
    print("frame", i, "launches", _lib.LAUNCHES - l0)
from torch.profiler import ProfilerActivity, profile
torch.cuda.synchronize()
ops.CONV_TRACE = []
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    trk.track_tensor(frames[1:2])
    torch.cuda.synchronize()
trace, ops.CONV_TRACE = ops.CONV_TRACE, None
rows = [(e.key, e.count, e.device_time_total) for e in prof.key_averages() if e.device_time_total > 0]
total = sum(r[2] for r in rows)
kern = sum(r[2] for r in rows if not r[0].startswith(("Memcpy", "Memset")))

# the same frame as one CUDA graph, input already in device memory (as bench.py replays it)
trg = UnicornSOTTrack(eng, (H, W), use_graph=True)
trg.initialize_tensor(frames[0:1], boxes[0, 0])
for _ in range(3):
    trg.track_tensor(frames[1:2])
c = trg._ctxs[0]
dev_frame = frames[1:2].to(eng.dev)
R = 20
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
c.stage(dev_frame)
torch.cuda.synchronize()
e0.record()
for _ in range(R):
    c.stage(dev_frame)
    c.graph.replay()
e1.record()
torch.cuda.synchronize()
step_ms = e0.elapsed_time(e1) / R

print(f"{torch.cuda.get_device_name()}: device time of one eager {H}x{W} frame {total / 1e3:.2f} ms in {sum(r[1] for r in rows)} "
      f"kernels and copies; kernels alone {kern / 1e3:.2f} ms; CUDA-graph step of the same frame {step_ms:.2f} ms")
for key, n, us in sorted(rows, key=lambda r: -r[2])[:20]:
    print(f"{us / 1e3:8.3f} ms {100 * us / total:5.1f} % {n:5d}x  {key[:110]}")

# per-layer convolutions: the conv kernels in start order are paired with the trace's launches in issue order; side branches run
# on their own streams, so each pairing is checked against the N tile in the kernel's template arguments
ck = sorted((e for e in prof.events() if "conv_gemm_kernel<" in e.name), key=lambda e: e.time_range.start)
if len(ck) != len(trace):
    print(f"conv table skipped: {len(ck)} conv kernels, {len(trace)} traced launches")
else:
    agg, mism = {}, 0
    for e, t in zip(ck, trace):
        bn, _, _, cl = [v.strip() for v in re.search(r"conv_gemm_kernel<([^>]*)>", e.name).group(1).split(",")][:4]
        code = int(bn) + (1000 if cl == "2" else 0)
        mism += bool(t["bn"]) and t["bn"] != code
        key = (t["M"], t["N"], t["K"], t["k"], t["s"], code, t["act"], t["gn"])
        a = agg.setdefault(key, [0, 0.0])
        a[0] += 1
        a[1] += e.time_range.elapsed_us()
    tot = sum(a[1] for a in agg.values())
    print(f"{len(ck)} conv launches, {tot / 1e3:.2f} ms ({100 * tot / kern:.1f} % of the kernel time)"
          + (f"; {mism} pairings disagree with the requested block_n" if mism else ""))
    print(f"{'M':>6} {'N':>5} {'K':>5} k s {'bn':>4} act gn   n  us/launch  TFLOP/s  share")
    for key, (n, us) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        M, N, K, k, s, bn, act, gn = key
        print(f"{M:6d} {N:5d} {K:5d} {k} {s} {bn:4d} {act:3d} {gn:2d} {n:3d} {us / n:10.1f} {2.0 * M * N * K * n / us / 1e6:8.1f} {100 * us / tot:5.1f}%")
if os.environ.get("UC_CONV_TRACE"):
    import json
    json.dump(trace, open(os.environ["UC_CONV_TRACE"], "w"))
if len(args) > 2:
    eng.save_tuning(args[2])
    print("saved tuning table", args[2], len(eng._bn_cache))
