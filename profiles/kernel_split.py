"""Per-kernel device time of one graph-replayed node-API job (LanPaint_KSampler.sample, the bench's flagship call).

torch.profiler (CUPTI activity records) around single jobs after warm-up (eager -> capture -> replay); the kernels
of the sampler loop are grouped by name and reported as launches per job, device us per job and share of the loop,
together with the card's name and power limit.

    python profiles/kernel_split.py --requests 128 [--rng torch] [--jobs 3]
"""
import argparse
import collections
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

import minicomfy  # noqa: E402

minicomfy.install()
from lanpaint_b200 import comfy_nodes as N  # noqa: E402
from lanpaint_b200.runner import SynthCondNet  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--requests", type=int, default=128)
ap.add_argument("--rng", default="torch")
ap.add_argument("--jobs", type=int, default=3)
args = ap.parse_args()
dev = torch.device("cuda:0")
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:  # noqa: BLE001
    card = f"nvidia-smi unavailable ({e})"
print(f"# card: {card}")

R = args.requests
g = torch.Generator().manual_seed(0)
y = torch.randn(R, 4, 128, 128, generator=g)
noise_mask = (torch.rand(R, 1, 128, 128, generator=g) < 0.5).float()
patcher = minicomfy.ModelPatcher(minicomfy.BaseModel(SynthCondNet()), dev)
patcher.model_options["lanpaint_b200"] = {"rng": args.rng}
node = N.LanPaint_KSampler()


def call(seed):
    with torch.no_grad():
        return node.sample(patcher, seed, 20, 5.0, "euler", "karras", 0.3, -0.2,
                           {"samples": y, "noise_mask": noise_mask}, 1.0, 5, "Image First", "", N.IMAGE_MODE)


for k in range(4):
    call(k)
torch.cuda.synchronize()
tot = collections.defaultdict(lambda: [0, 0.0])
for j in range(args.jobs):
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call(100 + j)
        torch.cuda.synchronize()
    recs = [(e.name(), e.start_ns() / 1e3, e.duration_ns() / 1e3) for e in prof.profiler.kineto_results.events()
            if str(e.device_type()).endswith("CUDA") and e.duration_ns() > 0]
    lp = [r for r in recs if "lp::" in r[0]]
    t0 = min(s for _, s, _ in lp)
    t1 = max(s + d for _, s, d in lp)
    for n, s, d in recs:
        if s >= t0 and s + d <= t1:
            key = n.split("(")[0]
            tot[key][0] += 1
            tot[key][1] += d
    print(f"# job {j}: span {t1 - t0:.1f} us, mode={N.LAST_RUN['mode']}")
loop = sum(v[1] for v in tot.values()) / args.jobs
print(f"# R={R} rng={args.rng}: kernel time per job {loop:.1f} us")
print("# launches/job   us/job   share   kernel")
for n, (c, d) in sorted(tot.items(), key=lambda kv: -kv[1][1]):
    print(f"{c / args.jobs:13.1f} {d / args.jobs:8.1f} {100 * d / args.jobs / loop:6.2f}%   {n[:150]}")
