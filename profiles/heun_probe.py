"""heun through the fused sampler loop against its two other routes, and the new step-boundary kernel per launch
(DESIGN §4).

Part 1: `LanPaint_KSampler.sample` (heun, karras-20, N = 5, the synthetic network, ComfyUI's callback) at R = 8 and
R = 128, three routes alternated in one process: fused (option "fused_heun"), the whole-sampler graph (the default
options) and per-sigma ("fused_sampler" and "sampler_graph" off).  Each arm is warmed until its graphs replay, then timed with device
events around enough jobs for >= --min-seconds of device work, three alternations.  "deferred_max_ms" is raised so
that the whole-sampler graph takes these short jobs.
Part 2: the same three routes with minicomfy.networks.DiTStandIn ([1,16,128,128], flow, simple-20) and default
options: a real network's job is too long for deferred callbacks, so the callback is live (per-step graphs on the
fused route) and the whole-sampler graph gives up, leaving the per-sigma route.
Part 3, as profiles/ancestral_probe.py: on job-shaped R = 128 operands, the cond + uncond network calls, then ONE
boundary launch timed alone between two events, three operand sets cycled: lp_boundary_known (boundary_kernel, the
Euler boundary) next to lp_boundary_midpoint as heun's predictor (x -> x2, writes out, call B's replace step) and
lp_boundary_heun as its corrector (x, x2 and the predictor's out -> x, no out, the next step's replace step), as the
fused job launches them.  Prints the card and its power limit with the numbers.

    python profiles/heun_probe.py [--requests 8,128] [--min-seconds 1.0] [--rounds 30] [--no-dit]
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

import minicomfy  # noqa: E402
from lanpaint_b200 import _native  # noqa: E402
from lanpaint_b200.engine import pack_known, pack_mask  # noqa: E402
from lanpaint_b200.runner import SynthCondNet, times_from_sigma  # noqa: E402
from lanpaint_b200.schedule import Hyper, build_table  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--requests", default="8,128")
ap.add_argument("--min-seconds", type=float, default=1.0)
ap.add_argument("--rounds", type=int, default=30)
ap.add_argument("--no-dit", action="store_true")
args = ap.parse_args()
assert torch.cuda.is_available(), "the probe measures on a CUDA device"
dev = torch.device("cuda:0")
try:
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30).stdout.strip()
except Exception as e:  # noqa: BLE001
    card = f"nvidia-smi unavailable ({e})"
print(f"# card: {card}")

minicomfy.install()
from lanpaint_b200 import comfy_nodes as N  # noqa: E402

ROUTES = {"fused": {"fused_heun": True}, "sampler-graph": {},
          "per-sigma": {"fused_sampler": False, "sampler_graph": False}}


def node_arm(base, shape, route, extra, scheduler, cfg):
    patcher = minicomfy.ModelPatcher(base, dev)
    patcher.model_options["lanpaint_b200"] = dict(ROUTES[route], **extra)
    g = torch.Generator().manual_seed(shape[0])
    latent = {"samples": torch.randn(shape, generator=g),
              "noise_mask": (torch.rand((shape[0], 1) + shape[2:], generator=g) < 0.5).float()}

    def job():
        with torch.no_grad():
            N.LanPaint_KSampler().sample(patcher, 7, 20, cfg, "heun", scheduler, 0.3, -0.2, latent, 1.0, 5,
                                         "Image First", "", N.IMAGE_MODE)
    return job


def time_jobs(job, min_seconds):
    """-> (ms of device time per job between two events around `n` back-to-back node calls, n)."""
    n, total = 1, 0.0
    while True:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            job()
        e1.record()
        e1.synchronize()
        total = e0.elapsed_time(e1)
        if total >= 1e3 * min_seconds:
            return total / n, n
        n = max(n + 1, int(n * 1.2e3 * min_seconds / max(total, 1e-3)))


def compare(label, arms):
    for name, job in arms.items():
        for _ in range(4):      # eager (and the recorded job), capture, replay
            job()
        print(f"# {label} {name}: LAST_RUN mode {N.LAST_RUN['mode']!r}, fused {N.LAST_RUN['fused']}")
    torch.cuda.synchronize()
    for alt in range(3):
        row = []
        for name, job in arms.items():
            ms, n = time_jobs(job, args.min_seconds)
            row.append(f"{name} {ms:9.2f} ms/job (n={n})")
        print(f"{label}, alternation {alt}: " + " | ".join(row))
    N._ENGINES.clear()


# ---- part 1: whole node calls, synthetic network ------------------------------------------------------------------
for R in (int(v) for v in args.requests.split(",")):
    base = minicomfy.BaseModel(SynthCondNet())
    compare(f"R={R} heun karras-20 N=5 synthetic",
            {r: node_arm(base, (R, 4, 128, 128), r, {"deferred_max_ms": 1e9}, "karras", 5.0) for r in ROUTES})

# ---- part 2: the DiT stand-in, live callback ------------------------------------------------------------------------
if not args.no_dit:
    from minicomfy.networks import DiTStandIn
    torch.manual_seed(1234)
    base = minicomfy.BaseModel(DiTStandIn().to(dev).eval(), model_type=minicomfy.ModelType.FLUX, latent_channels=16,
                               shift=1.15)
    compare("R=1 heun simple-20 N=5 DiT stand-in, live callback",
            {r: node_arm(base, (1, 16, 128, 128), r, {}, "simple", 1.0) for r in ROUTES})

# ---- part 3: one boundary launch after two network calls -----------------------------------------------------------
lib = _native.load()
P = C.c_void_p
R, SHAPE = 128, (4, 128, 128)
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
    sets.append(dict(y=y, nz=nz, pm=pm, dims=dims, kn=pack_known(pm, dims, y, nz),
                     x=torch.randn((R,) + SHAPE, generator=g).to(dev), out=torch.empty_like(y),
                     x2=torch.randn((R,) + SHAPE, generator=g).to(dev),
                     hc=torch.empty_like(y), hu=torch.empty_like(y)))
torch.cuda.synchronize()
pred, corr = _native.Midpoint(2.0, -0.6), _native.Heun(2.0, 1.4, -0.6)


def network(o):
    for h, coef in ((o["hc"], net_coef[0]), (o["hu"], net_coef[1])):
        _native.check(lib.lp_synth_denoiser_f32(P(o["x"].data_ptr()), P(h.data_ptr()), None, n_el, coef, stream), "net")


def heads(o):
    return _native.Heads(o["hc"].data_ptr(), o["hu"].data_ptr(), 0, 1, 5.0, 5.0)


def euler(o):
    hd = heads(o)
    return lib.lp_boundary_known(C.byref(hd), P(o["y"].data_ptr()), P(o["nz"].data_ptr()), P(o["pm"].data.data_ptr()),
                                 C.byref(o["kn"].struct), P(o["x"].data_ptr()), P(o["out"].data_ptr()), C.c_float(-0.1),
                                 P(tab.data_ptr()), C.byref(o["dims"]), stream)


def predictor(o):
    hd = heads(o)
    return lib.lp_boundary_midpoint(C.byref(hd), P(o["y"].data_ptr()), P(o["nz"].data_ptr()),
                                    P(o["pm"].data.data_ptr()), C.byref(o["kn"].struct), P(o["x"].data_ptr()),
                                    P(o["x"].data_ptr()), P(o["x2"].data_ptr()), P(o["out"].data_ptr()), C.byref(pred),
                                    P(tab.data_ptr()), C.byref(o["dims"]), stream)


def corrector(o):
    hd = heads(o)
    return lib.lp_boundary_heun(C.byref(hd), P(o["y"].data_ptr()), P(o["nz"].data_ptr()), P(o["pm"].data.data_ptr()),
                                C.byref(o["kn"].struct), P(o["x"].data_ptr()), P(o["x2"].data_ptr()),
                                P(o["out"].data_ptr()), None, C.byref(corr), P(tab.data_ptr()), C.byref(o["dims"]),
                                stream)


kernels = {"boundary_kernel (euler, packed, cfg, next)": euler,
           "boundary_midpoint_kernel (predictor, packed)": predictor,
           "boundary_heun_kernel (corrector, packed)": corrector}
res = {k: [] for k in kernels}
for rnd in range(args.rounds + 2):           # the first two rounds warm every kernel up and are dropped
    for name, launch in kernels.items():
        for o in sets:
            network(o)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _native.check(launch(o), name)
            e1.record()
            e1.synchronize()
            if rnd >= 2:
                res[name].append(1e3 * e0.elapsed_time(e1))
print(f"# R=128: median us per boundary launch right after the cond + uncond network calls "
      f"({3 * args.rounds} launches each; [p10, p90]); all but the corrector write `out`")
for name, t in res.items():
    t = sorted(t)
    n = len(t)
    print(f"{name:50s} {t[n // 2]:8.1f} [{t[n // 10]:5.1f},{t[(9 * n) // 10]:5.1f}]")
