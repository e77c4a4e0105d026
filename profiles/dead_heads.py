"""Dead heads: what discarding the network's output from the L2 (LP_HEADS_DEAD, DESIGN §4) saves per update launch.

Per repetition, on job-shaped R = 128 operands, in the form of profiles/l2_handoff.py: the two network calls a node
makes (cond, then uncond: lp_synth_denoiser_f32 reads x and writes one head, front to back), then ONE update launch
with its heads flagged dead, timed alone between two CUDA events, then the next cond network call, timed on its own
(it rewrites the discarded head; without the discard it competes with the write-back of the dirty lines).  Three
operand sets are cycled, as in runner.time_steady_substep.  Option "discard_heads" 0 | 1 is interleaved in each
round.  Kernels: the steady torch-stream TMA sub-step (packed known operands, the node default), the philox TMA
sub-step, the packed LDG boundary, the torch-stream TMA ancestral boundary.  Prints the card, its power limit and a
table of median us per launch.

    python profiles/dead_heads.py [--requests 128] [--rounds 30]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from lanpaint_b200 import _native  # noqa: E402
from lanpaint_b200.engine import _DrawPlan, pack_known, pack_mask  # noqa: E402
from lanpaint_b200.runner import times_from_sigma  # noqa: E402
from lanpaint_b200.schedule import Hyper, build_table  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--requests", type=int, default=128)
ap.add_argument("--rounds", type=int, default=30)
args = ap.parse_args()
settings = (0, 1)
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
anc = _native.Ancestral(sigma, -0.3, 1.0, 0.5)
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


def net_call(o, which):
    h = o["hc"] if which == 0 else o["hu"]
    rc = lib.lp_synth_denoiser_f32(P(o["x"].data_ptr()), P(h.data_ptr()), None, n_el, net_coef[which], stream)
    _native.check(rc, "lp_synth_denoiser_f32")


def heads(o):  # raw cond / uncond, combined in the update kernel, flagged dead
    return _native.Heads(o["hc"].data_ptr(), o["hu"].data_ptr(), _native.DTYPE_F32 | _native.HEADS_DEAD, 1, 5.0, 5.0)


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


def ancestral(o):
    r = plans["torch"].rng_struct(1)
    hd = heads(o)
    return lib.lp_boundary_ancestral(C.byref(hd), P(o["y"].data_ptr()), P(o["nz"].data_ptr()),
                                     P(o["pm"].data.data_ptr()), C.byref(o["kn"].struct), P(o["x"].data_ptr()),
                                     P(o["out"].data_ptr()), C.byref(anc), C.byref(r), P(tab.data_ptr()),
                                     C.byref(o["dims"]), stream)


kernels = {"torch TMA sub-step (packed, steady)": torch_substep, "philox TMA sub-step (steady, merged)": philox_substep,
           "LDG boundary (packed, cfg, euler, next)": boundary, "torch TMA ancestral boundary (packed, cfg)": ancestral}
upd = {(k, v): [] for k in kernels for v in settings}
cond = {(k, v): [] for k in kernels for v in settings}
for rnd in range(args.rounds + 2):           # the first two rounds warm every shape up and are dropped
    for name, launch in kernels.items():
        for v in settings:
            assert lib.lp_set_option(b"discard_heads", v) == 0
            for o in sets:
                net_call(o, 0)
                net_call(o, 1)
                ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                ev[0].record()
                _native.check(launch(o), name)
                ev[1].record()
                net_call(o, 0)
                ev[2].record()
                ev[2].synchronize()
                if rnd >= 2:
                    upd[(name, v)].append(1e3 * ev[0].elapsed_time(ev[1]))
                    cond[(name, v)].append(1e3 * ev[1].elapsed_time(ev[2]))
lib.lp_set_option(b"discard_heads", 1)


def stat(t):
    t = sorted(t)
    n = len(t)
    return t[n // 2], t[n // 10], t[(9 * n) // 10]


print(f"# R={R}: median us per launch ({3 * args.rounds} launches each; [p10, p90]); update = the launch right after "
      "the cond + uncond network calls, cond = the network call right after it")
print(f"{'kernel':44s}{'update, keep':>24s}{'update, discard':>24s}{'saved':>8s}{'cond, keep':>24s}"
      f"{'cond, discard':>24s}{'saved':>8s}")
for name in kernels:
    cells = []
    for res in (upd, cond):
        m = [stat(res[(name, v)]) for v in settings]
        cells += [f"{a:8.1f} [{b:5.1f},{c:5.1f}]" for a, b, c in m] + [f"{m[0][0] - m[1][0]:6.1f}"]
    print(f"{name:44s}" + "".join(f"{c:>24s}" if i % 3 != 2 else f"{c:>8s}" for i, c in enumerate(cells)))
