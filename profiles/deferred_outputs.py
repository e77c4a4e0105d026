"""Deferred outputs: what storing the denoised latent `out` costs the fused Euler loop's step-boundary launch.

Per repetition, on job-shaped R = 128 operands, in the form of profiles/dead_heads.py: the two network calls a node
makes (cond, then uncond: lp_synth_denoiser_f32 reads x and writes one head), then ONE packed LDG boundary launch
(lp_boundary_known_rows: CFG combine, Euler update, next replace step, heads flagged dead), timed alone between two
CUDA events.  Three operand sets are cycled.  The `out` store is interleaved in each round as: every row (what each
outer step of a deferred job stored for any callback), row 0 only (out_rows = 1, "preview") and none (out_rows = 0,
"final").  The byte count predicts the saving: the boundary moves 24.25 B per element with `out` and 20.25 without,
so a launch at the copy rate takes about 4/24.25 = 16.5 % less time.  Prints the card, its power limit and a table of
median us per launch.

    python profiles/deferred_outputs.py [--requests 128] [--rounds 30]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from lanpaint_b200 import _native  # noqa: E402
from lanpaint_b200.engine import pack_known, pack_mask  # noqa: E402
from lanpaint_b200.runner import times_from_sigma  # noqa: E402
from lanpaint_b200.schedule import Hyper, build_table  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--requests", type=int, default=128)
ap.add_argument("--rounds", type=int, default=30)
args = ap.parse_args()
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
s = torch.full((R,), 2.0, dtype=torch.float32)
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
    sets.append(dict(y=y, nz=nz, pm=pm, dims=dims, kn=kn, x=x, out=torch.empty_like(x), hc=torch.empty_like(x),
                     hu=torch.empty_like(x)))
torch.cuda.synchronize()


def net_call(o, which):
    h = o["hc"] if which == 0 else o["hu"]
    rc = lib.lp_synth_denoiser_f32(P(o["x"].data_ptr()), P(h.data_ptr()), None, n_el, net_coef[which], stream)
    _native.check(rc, "lp_synth_denoiser_f32")


def boundary(o, rows):
    hd = _native.Heads(o["hc"].data_ptr(), o["hu"].data_ptr(), _native.DTYPE_F32 | _native.HEADS_DEAD, 1, 5.0, 5.0)
    return lib.lp_boundary_known_rows(C.byref(hd), P(o["y"].data_ptr()), P(o["nz"].data_ptr()),
                                      P(o["pm"].data.data_ptr()), C.byref(o["kn"].struct), P(o["x"].data_ptr()),
                                      P(o["out"].data_ptr()), rows, C.c_float(-0.1), P(tab.data_ptr()),
                                      C.byref(o["dims"]), stream)


settings = {"out, every row": R, "out, row 0 (preview)": 1, "no out (final)": 0}
upd = {k: [] for k in settings}
for rnd in range(args.rounds + 2):           # the first two rounds warm every shape up and are dropped
    for name, rows in settings.items():
        for o in sets:
            net_call(o, 0)
            net_call(o, 1)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            ev[0].record()
            _native.check(boundary(o, rows), name)
            ev[1].record()
            ev[1].synchronize()
            if rnd >= 2:
                upd[name].append(1e3 * ev[0].elapsed_time(ev[1]))


def stat(t):
    t = sorted(t)
    n = len(t)
    return t[n // 2], t[n // 10], t[(9 * n) // 10]


full = stat(upd["out, every row"])[0]
print(f"# R={R}: median us per boundary launch right after the cond + uncond network calls "
      f"({3 * args.rounds} launches each; [p10, p90]); predicted saving without out: {100 * 4 / 24.25:.1f} %")
print(f"{'setting':24s}{'us':>24s}{'saved':>10s}")
for name in settings:
    m, lo, hi = stat(upd[name])
    print(f"{name:24s}{f'{m:8.1f} [{lo:6.1f},{hi:6.1f}]':>24s}{f'{100 * (full - m) / full:8.1f} %':>10s}")
