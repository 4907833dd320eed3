"""Run init + N eager (non-graph) SOT frames of a config, then print where the device time of one more frame goes: per-kernel
device time from torch.profiler (CUDA activities), grouped by kernel name, largest first.

usage: profile_frame.py [config] [frames] [tuning table to save]"""
import os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from unicorn_b200 import _lib, ops
from unicorn_b200.engine import UnicornEngine
from unicorn_b200.sot import UnicornSOTTrack
from unicorn_b200.synthetic import make_video
from unicorn_b200.weights import make_state_dict
name = sys.argv[1] if len(sys.argv) > 1 else "unicorn_track_large"
nfr = int(sys.argv[2]) if len(sys.argv) > 2 else 2
H, W = (320, 320) if "tiny" in name else (800, 1280)
sd = make_state_dict(name, 0)
frames, boxes = make_video(nfr + 1, H, W, seed=0)
eng = UnicornEngine(sd, name)
trk = UnicornSOTTrack(eng, (H, W), use_graph=False)
trk.initialize_tensor(frames[0:1], boxes[0, 0])
print("launches after init", _lib.LAUNCHES)
for i in range(nfr):
    l0 = _lib.LAUNCHES
    ops.CONV_TRACE = [] if i == nfr - 1 else None
    trk.track_tensor(frames[1 + i:2 + i])
    print("frame", i, "launches", _lib.LAUNCHES - l0)
from torch.profiler import ProfilerActivity, profile
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    trk.track_tensor(frames[1:2])
    torch.cuda.synchronize()
rows = [(e.key, e.count, e.device_time_total) for e in prof.key_averages() if e.device_time_total > 0]
total = sum(r[2] for r in rows)
print(f"{torch.cuda.get_device_name()}: device time of one eager {H}x{W} frame {total / 1e3:.2f} ms in {sum(r[1] for r in rows)} kernels")
for key, n, us in sorted(rows, key=lambda r: -r[2])[:20]:
    print(f"{us / 1e3:8.3f} ms {100 * us / total:5.1f} % {n:5d}x  {key[:110]}")
if os.environ.get("UC_CONV_TRACE"):
    import json
    json.dump(ops.CONV_TRACE, open(os.environ["UC_CONV_TRACE"], "w"))
if len(sys.argv) > 3:
    eng.save_tuning(sys.argv[3])
    print("saved tuning table", sys.argv[3], len(eng._bn_cache))
