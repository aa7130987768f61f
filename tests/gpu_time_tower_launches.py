"""Times the DownSample tower launch by launch: a torch.profiler table of every kernel one initial_inference call launches
(median over the profiled calls, per position in the launch order), then uninstrumented initial_inference medians with CUDA
events, at B = 1024 (DBG_B) for 84, 96 and 64 px frames (DBG_PX="84,96,64").  Prints the card name and power limit it ran
on.  LZ_LIB_TAG=<tag> picks lightzero_b200/_lib/<tag>/liblzb200.so (see _build.py), so one GPU session can compare builds."""
import os
import subprocess
import sys

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lightzero_b200 as lzb
from lightzero_b200.synthetic_weights import synthetic_state_dict

B, A = int(os.environ.get("DBG_B", 1024)), 18
PXS = [int(v) for v in os.environ.get("DBG_PX", "84,96,64").split(",")]
NPROF, NTIME = 10, 15


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def median(v):
    v = sorted(v)
    return v[len(v) // 2]


def launch_table(model, obs):
    for _ in range(3):
        model.initial_inference(obs)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(NPROF):
            model.initial_inference(obs)
        torch.cuda.synchronize()
    kern = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower()
                   and "memset" not in e.name.lower()), key=lambda e: e.time_range.start)
    calls = []                                  # each call starts with the stem launch; a one-off launch makes a call longer
    for e in kern:
        if "stem" in e.name or not calls:
            calls.append([])
        calls[-1].append(e)
    n = median([len(c) for c in calls])
    calls = [c for c in calls if len(c) == n]
    return [(calls[0][i].name, median([c[i].time_range.elapsed_us() for c in calls])) for i in range(n)]


def time_initial(model, obs):
    ms = []
    for i in range(NTIME + 3):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        model.initial_inference(obs[i % len(obs)])
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return median(ms[3:]), min(ms[3:])


print(f"card: {card()}  lib tag: {os.environ.get('LZ_LIB_TAG', '-')}  B={B}")
for px in PXS:
    model = lzb.MuZeroModel(observation_shape=(4, px, px), action_space_size=A, downsample=True).load_state_dict(synthetic_state_dict((4, px, px), A))
    obs = [torch.rand(B, 4, px, px).cuda() for _ in range(3)]
    rows = launch_table(model, obs[0])
    print(f"--- {px} px: per-launch median of {NPROF} profiled calls (us)")
    for name, us in rows:
        print(f"  {us:9.1f}  {name[:110]}")
    print(f"  {sum(us for _, us in rows):9.1f}  (sum of kernel times)")
    med, mn = time_initial(model, obs)
    print(f"{px} px initial_inference B={B}: median {med:.3f} ms, min {mn:.3f} ms (CUDA events, {NTIME} calls, profiler off)")
    del model, obs
    torch.cuda.empty_cache()
