"""The L2 hand-off from the network to the update kernels (DESIGN §4, option "l2_handoff").

Per repetition, on job-shaped R = 128 operands: the two network calls a node makes (cond, then uncond:
lp_synth_denoiser_f32 reads x and writes one head, front to back), then ONE update launch timed alone between two
CUDA events.  Three operand sets are cycled, as in runner.time_steady_substep, so nothing but what the network
calls just touched can be in L2.  Kernels: the steady torch-stream TMA sub-step (packed known operands, the node
default), the philox TMA sub-step, the packed LDG boundary.  Every "l2_handoff" setting is interleaved in each round.
Prints the card, its power limit, a table of median us per update launch, and the L2-cold steady-sub-step figure of
runner.time_steady_substep for comparison.

    python profiles/l2_handoff.py [--requests 128] [--rounds 30] [--settings 0,1,2,3]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from lanpaint_b200 import _native  # noqa: E402
from lanpaint_b200.engine import LanPaint, _DrawPlan, pack_known, pack_mask  # noqa: E402
from lanpaint_b200.runner import SynthDenoiser, VESampling, time_steady_substep, times_from_sigma  # noqa: E402
from lanpaint_b200.schedule import Hyper, build_table  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--requests", type=int, default=128)
ap.add_argument("--rounds", type=int, default=30)
ap.add_argument("--settings", default="0,1,2,3", help="l2_handoff values: bit 1 tail-first, bit 2 evict-first")
args = ap.parse_args()
settings = [int(v) for v in args.settings.split(",")]
dev = torch.device("cuda:0")
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:  # noqa: BLE001
    card = f"nvidia-smi unavailable ({e})"
print(f"# card: {card}")

lib = _native.load()
P = C.c_void_p
R, SHAPE = args.requests, (4, 128, 128)
n_el = R * 4 * 128 * 128
stream = P(torch.cuda.current_stream(dev).cuda_stream)
g = torch.Generator().manual_seed(0)
per_row, spatial = 4 * 128 * 128, 128 * 128
sigma = 2.0
s = torch.full((R,), sigma, dtype=torch.float32)
ve, abt, _ = times_from_sigma(s, False)
tab = torch.from_numpy(build_table(abt.numpy(), ve.numpy(), Hyper(0.2, 5.0, 1.0, 1.0, False))).to(dev)
net_coef = [(C.c_float * 5)(0.7, 0.1, c, 0.0, 0.0) for c in (0.05, -0.05)]   # cond, uncond
sets = []
for r in range(3):
    y = torch.randn((R,) + SHAPE, generator=g).to(dev)
    nz = torch.randn((R,) + SHAPE, generator=g).to(dev)
    pm = pack_mask((torch.rand((R, 1) + SHAPE[1:], generator=g) < 0.5).to(dev), y)
    dims = _native.Dims(R, per_row, spatial, pm.row_stride, pm.channel_stride)
    kn = pack_known(pm, dims, y, nz)
    x = torch.randn((R,) + SHAPE, generator=g).to(dev)
    sets.append(dict(y=y, nz=nz, pm=pm, dims=dims, kn=kn, x=x, c=torch.randn_like(x), out=torch.empty_like(x),
                     hc=torch.empty_like(x), hu=torch.empty_like(x)))
torch.cuda.synchronize()


def network(o):
    for h, coef in ((o["hc"], net_coef[0]), (o["hu"], net_coef[1])):
        rc = lib.lp_synth_denoiser_f32(P(o["x"].data_ptr()), P(h.data_ptr()), None, n_el, coef, stream)
        _native.check(rc, "lp_synth_denoiser_f32")


def heads(o):
    return _native.Heads(o["hc"].data_ptr(), o["hu"].data_ptr(), 0, 1, 5.0, 5.0)


plans = {"torch": _DrawPlan("torch", sets[0]["x"], 1 << 20), "philox": _DrawPlan("philox", sets[0]["x"], 1 << 20)}


def torch_substep(o):
    r = plans["torch"].rng_struct(2)
    hd = heads(o)
    return lib.lp_substep_known(P(o["x"].data_ptr()), C.byref(hd), P(o["y"].data_ptr()), P(o["pm"].data.data_ptr()),
                                C.byref(o["kn"].struct), P(o["c"].data_ptr()), None, None, P(tab.data_ptr()),
                                C.byref(o["dims"]), C.byref(r), _native.SUBSTEP_FUSE_NEXT, stream)


def philox_substep(o):
    r = plans["philox"].rng_struct(1)
    hd = heads(o)
    return lib.lp_substep(P(o["x"].data_ptr()), C.byref(hd), P(o["y"].data_ptr()), P(o["pm"].data.data_ptr()),
                          P(o["c"].data_ptr()), None, None, P(tab.data_ptr()), C.byref(o["dims"]), C.byref(r),
                          _native.SUBSTEP_FUSE_NEXT | _native.SUBSTEP_MERGE_NOISE, stream)


def boundary(o):
    hd = heads(o)
    return lib.lp_boundary_known(C.byref(hd), P(o["y"].data_ptr()), P(o["nz"].data_ptr()), P(o["pm"].data.data_ptr()),
                                 C.byref(o["kn"].struct), P(o["x"].data_ptr()), P(o["out"].data_ptr()), C.c_float(-0.1),
                                 P(tab.data_ptr()), C.byref(o["dims"]), stream)


kernels = {"torch TMA sub-step (packed, steady)": torch_substep, "philox TMA sub-step (steady, merged)": philox_substep,
           "LDG boundary (packed, cfg, euler, next)": boundary}
res = {(k, v): [] for k in kernels for v in settings}
for rnd in range(args.rounds + 2):           # the first two rounds warm every shape up and are dropped
    for name, launch in kernels.items():
        for v in settings:
            assert lib.lp_set_option(b"l2_handoff", v) == 0
            for o in sets:
                network(o)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                _native.check(launch(o), name)
                e1.record()
                e1.synchronize()
                if rnd >= 2:
                    res[(name, v)].append(1e3 * e0.elapsed_time(e1))
lib.lp_set_option(b"l2_handoff", 3)

print(f"# R={R}: median us per update launch right after the cond + uncond network calls "
      f"({3 * args.rounds} launches each; [p10, p90])")
print("# setting: 0 head-first | 1 tail-first | 2 head-first + evict-first | 3 tail-first + evict-first (default)")
print(f"{'kernel':42s}" + "".join(f"{v:>22d}" for v in settings))
for name in kernels:
    row = []
    for v in settings:
        t = sorted(res[(name, v)])
        n = len(t)
        row.append(f"{t[n // 2]:8.1f} [{t[n // 10]:5.1f},{t[(9 * n) // 10]:5.1f}]")
    print(f"{name:42s}" + "".join(f"{c:>22s}" for c in row))

eng = LanPaint(SynthDenoiser(VESampling()), NSteps=5, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2,
               MinStepFrac=1.0, rng="torch", batched_replace="per_sample")
for v in settings:
    lib.lp_set_option(b"l2_handoff", v)
    cold = sorted(time_steady_substep(eng, sets[0]["y"], sets[0]["pm"], sigma=2.0, launches=53, repeats=20, rotate=3))
    print(f"# time_steady_substep (torch, dense, L2-cold burst of 53), l2_handoff={v}: "
          f"mean {sum(cold) / len(cold):.1f} us, median {cold[len(cold) // 2]:.1f} us")
lib.lp_set_option(b"l2_handoff", 3)
