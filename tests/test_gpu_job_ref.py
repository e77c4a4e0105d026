"""GPU: whole inpainting jobs against an fp64 restatement, at production sizes, with a network that couples positions.

The launch tests (tests/test_gpu_launch_ref.py) check every update kernel one launch at a time.  These check how the
job layer chains ~126 of them -- `runner.GraphedJob` (eager, per-step graphs, whole-job graph), `runner.SamplerGraphJob`,
the per-sigma graphs of the engine and the node glue around them -- against `_job_ref.job` in fp64: the same sampler
Python around `O.outer_step` (pinned to the reference by the node goldens), the schedule and the (VE, abt, flow t)
triple in fp32 as the node computes them, every Gaussian drawn as `torch.randn(shape, float32)` on the device's
default generator (the engine's torch stream, upcast).

The network is `_node_cases.mixing_denoiser`: with a pointwise one nothing a job does at known positions -- cfg_BIG,
lambda, the replace step and its next-step table, the packed noise image -- reaches the result
(tests/test_job_ref_host.py).  The latents are large enough (>= 2^18 elements) that the sub-steps run the kernels
production runs, and each case asserts which sub-step kernel that was.

Each case asserts: max|got - want| <= B * max|want| on the final latent and on every step's denoised latent (where
a callback exists), whose known positions must equal y bit for bit; and the generator offset after the job equals the
reference's."""
import collections
import json
import sys

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import _job_ref as J
import minicomfy
from _launch_ref import canon
from _node_cases import NEG, POS, mixing_denoiser
from oracle import langevin_oracle as O

pytestmark = pytest.mark.gpu

B = 4e-6    # max|got - want| / max|want|, final and per-step latents: 3.6x the worst measured on an H100 (DESIGN.md §6)
WORST = collections.defaultdict(float)   # case -> largest error seen


def _generator(dev):
    torch.cuda.init()           # the default generators exist once CUDA is initialised
    return torch.cuda.default_generators[dev.index]


def _rel(got, want):
    got = got.to(device=want.device, dtype=torch.float64)
    return float((got - want).abs().max() / want.abs().max())


def _check(case, label, got, want):
    err = _rel(got, want)
    WORST[case] = max(WORST[case], err)
    assert err <= B, f"{case} {label}: {err:.3g} > B = {B}"


def _check_steps(case, label, got_steps, want_steps, y, known):
    """Per-step denoised latents: the bound, and y at known positions bit for bit."""
    assert [i for i, _ in got_steps] == list(range(len(want_steps))), (case, label, [i for i, _ in got_steps])
    for (i, d), w in zip(got_steps, want_steps):
        _check(case, f"{label} denoised[{i}]", d, w)
        assert torch.equal(d[known], y[known]), f"{case} {label}: denoised[{i}] differs from y at a known position"


def _sub_kernels(fn):
    """Run fn() under torch.profiler -> (its result, the canonical names of the sub-step kernels it launched)."""
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    names = {canon(e.name()) for e in prof.profiler.kineto_results.events() if "lp::" in e.name()}
    return out, {n for n in names if n.startswith("substep")}


def _assert_torch_tma(case, names, packed):
    """Every sub-step launch ran the torch-stream TMA kernel, with packed (or dense) known operands."""
    assert names, f"{case}: no sub-step kernel recorded"
    bad = [n for n in names if not (n.startswith("substep_torch_tma_kernel<") and n.endswith(f",{int(packed)}>"))]
    assert not bad, (case, sorted(names))


def _blob(shape, gen):
    """1 (regenerate) inside an ellipsoid over the trailing axes, 0 around it."""
    axes = [torch.linspace(-1.0, 1.0, n) for n in shape[2:]]
    grids = torch.meshgrid(*axes, indexing="ij")
    c = [float(v) * 0.3 for v in torch.rand(len(grids), generator=gen) - 0.5]
    r = sum(((g - ci) / 0.6) ** 2 for g, ci in zip(grids, c))
    return (r < 1.0).float().reshape(shape)


def _mask(kind, shape, gen):
    """A LATENT noise_mask (1 = regenerate) at the latent's resolution."""
    B_, sp = shape[0], tuple(shape[2:])
    if kind == "rand":
        return (torch.rand((B_, 1) + sp, generator=gen) < 0.5).float()
    if kind == "rand1":         # one mask for the whole batch
        return (torch.rand((1, 1) + sp, generator=gen) < 0.5).float()
    if kind == "blob":
        return _blob((1, 1) + sp, gen)
    if kind == "free":
        return torch.ones((B_, 1) + sp)
    if kind == "known":
        return torch.zeros((B_, 1) + sp)
    raise KeyError(kind)


def _full(mask, shape):
    """The denoise mask the node hands the sampler for a mask at the latent's resolution, in image inpainting mode
    (video mode would widen it over a 5-frame window)."""
    return minicomfy.repeat_to_batch_size(mask, shape[0]).expand(shape)


def _recorder(store):
    """latent_preview.prepare_callback stand-in: keeps every step's denoised latent (a device copy, stream-ordered)."""
    def prepare_callback(model, steps, x0_output_dict=None):
        def callback(step, x0, x, total_steps):
            store.append((step, x0.detach().clone()))
        return callback
    return prepare_callback


# ---------------------------------------------------------------------------------------------------------------
# the node path: LanPaint_KSampler.sample
# ---------------------------------------------------------------------------------------------------------------
NODE = dict(shape=(8, 4, 128, 128), mask="rand", mode="Image First", steps=20, n=5, cfg=5.0, sampler="euler",
            scheduler="karras", model_type="EPS", shift=1.0, wan22=False, opts=None, calls=2,
            modes=None, packed=(True, True))
# packed: the operands the (first, last) call's sub-steps read.  The fused Euler loop (GraphedJob) and the
# whole-sampler graph (SamplerGraphJob) build the packed known-operand layout once per job; the per-sigma path
# (the engine behind k-diffusion's own loop, and the eager job a SamplerGraphJob records) reads the dense operands.
NODE_CASES = {}
for _m in ("rand", "rand1"):
    for _p in ("Image First", "Prompt First"):
        for _d in (True, False):
            NODE_CASES[f"b8-{_m}-{_p.split()[0].lower()}-{'deferred' if _d else 'steps'}"] = dict(
                NODE, mask=_m, mode=_p, calls=4, opts={"deferred_callbacks": _d, "deferred_max_ms": 1e9},
                modes=["eager"] + ["job" if _d else "steps"] * 3)
NODE_CASES.update({
    "cfg3-tma-min-n10": dict(NODE, shape=(4, 4, 128, 128), n=10),
    "cfg4-flux-simple": dict(NODE, shape=(1, 16, 128, 128), model_type="FLUX", shift=1.15, scheduler="simple",
                             cfg=3.5),
    "cfg5-wan-blob": dict(NODE, shape=(1, 16, 21, 80, 45), model_type="FLOW", shift=3.0, wan22=True,
                          scheduler="simple", mask="blob", mode="Prompt First"),
    "flagship-r128": dict(NODE, shape=(128, 4, 128, 128)),
    "b8-all-free": dict(NODE, mask="free"),
    "b8-all-known": dict(NODE, mask="known", mode="Prompt First"),
    "b8-per-sigma-graphs": dict(NODE, opts={"fused_sampler": False, "sampler_graph": False}, modes=[None, None],
                                packed=(False, False)),
    # graphs captured at first sight, each after a warm-up pass: per-step graphs, then the whole-job graph
    "b8-graph-after-0": dict(NODE, calls=3, opts={"graph_after": 0, "deferred_max_ms": 1e9},
                             modes=["steps", "steps", "job"]),
    "b8-heun-sampler-graph": dict(NODE, sampler="heun", steps=10, calls=3, opts={"deferred_max_ms": 1e9},
                                  modes=[None, "sampler-graph", "sampler-graph"], packed=(False, True)),
})


@pytest.mark.parametrize("case", list(NODE_CASES))
def test_ksampler_job_matches_fp64(case, cuda_device, monkeypatch):
    """Calls: the first launches eagerly, the second captures, the third replays; a fourth (where there is one)
    replays the same graphs with a new seed and a new mask."""
    c = NODE_CASES[case]
    minicomfy.install()
    from lanpaint_b200 import comfy_nodes as N
    N._ENGINES.clear()
    dev = cuda_device
    shape = c["shape"]
    base = (minicomfy.WAN22 if c["wan22"] else minicomfy.BaseModel)(
        mixing_denoiser, model_type=getattr(minicomfy.ModelType, c["model_type"]), latent_channels=shape[1],
        shift=c["shift"])
    patcher = minicomfy.ModelPatcher(base, dev)
    if c["opts"] is not None:
        patcher.model_options["lanpaint_b200"] = dict(c["opts"])
    store = []
    monkeypatch.setattr(sys.modules["latent_preview"], "prepare_callback", _recorder(store))
    flow = c["model_type"] in ("FLUX", "FLOW")
    sampling = O.FlowSampling() if flow else O.VESampling()
    sig = minicomfy.KSampler(patcher, c["steps"], dev, c["sampler"], c["scheduler"]).sigmas
    md = J.max_denoise(base.model_sampling, sig[0])
    cfg_big = 1.0 if c["model_type"] == "FLUX" else (c["cfg"] if c["mode"] == "Image First" else -0.5)
    hp = O.Hyper(n_steps=c["n"], min_step_frac=1.0, flow=flow)
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    y = torch.randn(shape, generator=g)
    mask = _mask(c["mask"], shape, g)
    gen = _generator(dev)
    modes = []
    for k in range(c["calls"]):
        seed = 40 + k // 3              # calls 0..2 repeat one request; the fourth is a new one on the same graphs
        if k == 3:
            y, mask = torch.randn(shape, generator=g), _mask(c["mask"], shape, g)
        store.clear()

        def call():
            (out,) = N.LanPaint_KSampler().sample(patcher, seed, c["steps"], c["cfg"], c["sampler"], c["scheduler"],
                                                  POS, NEG, {"samples": y, "noise_mask": mask}, 1.0, c["n"],
                                                  c["mode"], "", N.IMAGE_MODE)
            return out["samples"]
        if k in (0, c["calls"] - 1):
            got, kernels = _sub_kernels(call)
            _assert_torch_tma(f"{case} call {k}", kernels, c["packed"][0 if k == 0 else 1])
        else:
            got = call()
        modes.append(N.LAST_RUN["mode"])
        torch.cuda.synchronize()
        offset = gen.get_offset()
        got_steps = list(store)

        noise = minicomfy.prepare_noise(y, seed)      # ComfyUI's CPU noise image; re-seeds every generator like the node
        yd = y.to(dev, torch.float64)
        dm = _full(mask, shape).to(dev, torch.float64)
        want_steps = []
        model = J.Guider(mixing_denoiser, sampling, c["cfg"], cfg_big)
        want = J.job(J.SAMPLERS[c["sampler"]], model, yd, noise.to(dev, torch.float64), dm, sig, hp, max_denoise=md,
                     callback=lambda i, d: want_steps.append(d))
        assert gen.get_offset() == offset, f"{case} call {k}: generator offset differs from the reference's"
        _check(case, f"call {k} out", got, want)
        _check_steps(case, f"call {k}", got_steps, want_steps, y.to(dev), (_full(mask, shape) <= 0.5).to(dev))
    if c["modes"] is not None:
        assert modes == c["modes"], modes
    else:
        assert modes[0] == "eager" and all(m in ("job", "steps") for m in modes[1:]), modes
    N._ENGINES.clear()


# ---------------------------------------------------------------------------------------------------------------
# runner.GraphedJob driven directly (serving hosts)
# ---------------------------------------------------------------------------------------------------------------
class _DeviceGuider:
    """The node's fused-CFG guider protocol over the mixing network: raw cond / uncond plus both scales."""

    def __init__(self, cfg, cfg_big):
        from lanpaint_b200.runner import VESampling
        self.inner_model, self.model_sampling, self.cfg, self.cfg_big = self, VESampling(), cfg, cfg_big

    def __call__(self, x, t, model_options=None, seed=None):
        from lanpaint_b200.engine import CfgPair
        return CfgPair(mixing_denoiser(x, t, POS), mixing_denoiser(x, t, NEG), self.cfg, self.cfg_big)


def _direct_setup(dev, shape, cfg=5.0, cfg_big=-0.5):
    from lanpaint_b200.engine import LanPaint
    from lanpaint_b200.runner import HostSchedule, karras_sigmas
    sig = karras_sigmas(20)
    eng = LanPaint(_DeviceGuider(cfg, cfg_big), NSteps=5, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2,
                   MinStepFrac=1.0, rng="torch")
    return eng, HostSchedule(sig, shape[0], 5), torch.tensor(sig, dtype=torch.float32)


def _direct_want(y, noise, known, sig, dev, cfg=5.0, cfg_big=-0.5, callback=None):
    model = J.Guider(mixing_denoiser, O.VESampling(), cfg, cfg_big)
    dm = 1.0 - known.to(dev, torch.float64).expand(y.shape)
    return J.job(J.SAMPLERS["euler"], model, y.to(dev, torch.float64), noise.to(dev, torch.float64), dm, sig,
                 O.Hyper(n_steps=5, min_step_frac=1.0), max_denoise=False, callback=callback)


@pytest.mark.parametrize("fused_euler", [True, False])
def test_graphed_job_modes_match_fp64(fused_euler, cuda_device):
    """One GraphedJob, four requests: mode "eager", "steps" and "job" with a callback, then "job" without one
    (fused_euler=False: the Euler update as two torch kernels, no fused next replace step)."""
    from lanpaint_b200.engine import pack_mask
    from lanpaint_b200.runner import GraphedJob
    dev = cuda_device
    shape = (8, 4, 128, 128)
    case = f"graphed-job-{'fused' if fused_euler else 'unfused'}"
    eng, sched, sig = _direct_setup(dev, shape)
    job = GraphedJob(eng, sched, shape, dev, fused_euler=fused_euler)
    g = torch.Generator().manual_seed(77 + fused_euler)
    gen = _generator(dev)
    for k, mode in enumerate(("eager", "steps", "job", "job")):
        y = torch.randn(shape, generator=g).to(dev)
        noise = torch.randn(shape, generator=g).to(dev)
        known = (torch.rand((shape[0], 1) + shape[2:], generator=g) < 0.5).to(dev)
        steps = []
        cb = None if k == 3 else (lambda i, d, x, n: steps.append((i, d.clone())))
        torch.cuda.manual_seed(900 + k)

        def run():
            return job.run(y, noise, pack_mask(known, y), callback=cb, mode=mode)
        if k == 0:
            got, kernels = _sub_kernels(run)
            _assert_torch_tma(case, kernels, True)
        else:
            got = run()
        torch.cuda.synchronize()
        offset = gen.get_offset()
        torch.cuda.manual_seed(900 + k)
        want_steps = []
        want = _direct_want(y, noise, known, sig, dev, callback=None if cb is None else (lambda i, d: want_steps.append(d)))
        assert gen.get_offset() == offset, f"{case} {mode}: generator offset differs from the reference's"
        _check(case, f"{mode} out", got, want)
        if cb is not None:
            _check_steps(case, mode, steps, want_steps, y, known.expand(shape))


def test_graphed_job_two_lanes_with_device_noise(cuda_device):
    """bench.py's serving e2e: two GraphedJobs on two streams, requests alternating between them, noise=None (each
    lane draws its noise image on the device).  The reference draws each request's noise image and then its
    Langevin draws from the one default generator in submission order, so it also checks that a lane's noise draw
    and its reserved draws do not overlap the other lane's."""
    from lanpaint_b200.runner import GraphedJob
    dev = cuda_device
    shape = (8, 4, 128, 128)
    eng_sched = [_direct_setup(dev, shape) for _ in range(2)]
    sig = eng_sched[0][2]
    lanes = [{"job": GraphedJob(e, s, shape, dev), "stream": torch.cuda.Stream(device=dev)} for e, s, _ in eng_sched]
    g = torch.Generator().manual_seed(5)
    gen = _generator(dev)
    reqs = []
    torch.cuda.manual_seed(123)
    for k in range(4):
        ln = lanes[k % 2]
        y = torch.randn(shape, generator=g).pin_memory()
        m = (torch.rand((shape[0], 1) + shape[2:], generator=g) < 0.5).to(torch.uint8).pin_memory()
        ln["stream"].synchronize()
        with torch.cuda.stream(ln["stream"]):
            out = ln["job"].run(y, None, m.to(dev, non_blocking=True))
            reqs.append((y, m, out, ln["job"].noise.clone()))
    torch.cuda.synchronize()
    offset = gen.get_offset()
    torch.cuda.manual_seed(123)
    for k, (y, m, out, noise) in enumerate(reqs):
        want_noise = torch.randn(shape, device=dev)
        assert torch.equal(noise, want_noise), f"lane request {k}: noise image is not the stream's next draw"
        want = _direct_want(y, noise, m.bool(), sig, dev)
        _check("graphed-job-two-lanes", f"request {k}", out, want)
    assert gen.get_offset() == offset


def test_report_worst_errors():
    """Prints the largest max|got - want| / max|want| per case (final and per-step latents)."""
    if not WORST:
        pytest.skip("no job case ran")
    print("job-level max |got - fp64| / max|fp64| per case:", json.dumps(dict(sorted(WORST.items())), indent=1))
    assert max(WORST.values()) <= B
