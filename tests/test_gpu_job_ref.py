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
reference's.  Besides the plain Euler KSampler the node routes users reach are covered: a KSamplerAdvanced window
with leftover noise, add_noise = disable, denoise < 1, euler_ancestral, SamplerCustomAdvanced on Flux (both outputs),
an audio-video pack through `outer_sample(latent_shapes=...)` and the inner early stop."""
import collections
import json
import sys

import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import _job_ref as J
import minicomfy
from _launch_ref import canon
from _node_cases import NEG, POS, FixedNoise, av_shift_sigma, av_shift_slope, mixing_denoiser
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


def _lp_kernels(fn):
    """Run fn() under torch.profiler -> (its result, the canonical names of the library kernels it launched)."""
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, {canon(e.name()) for e in prof.profiler.kineto_results.events() if "lp::" in e.name()}


def _sub_kernels(fn):
    """Run fn() under torch.profiler -> (its result, the canonical names of the sub-step kernels it launched)."""
    out, names = _lp_kernels(fn)
    return out, {n for n in names if n.startswith("substep")}


def _assert_torch_tma(case, names, packed):
    """Every sub-step launch ran the torch-stream TMA kernel, with packed (or dense) known operands."""
    assert names, f"{case}: no sub-step kernel recorded"
    bad = [n for n in names if not (n.startswith("substep_torch_tma_kernel<") and n.endswith(f",{int(packed)}>"))]
    assert not bad, (case, sorted(names))


def _assert_family(case, names, family):
    """Every sub-step launch ran one kernel family (a side output or a row split rules the TMA kernels out)."""
    subs = {n for n in names if n.startswith("substep")}
    assert subs, f"{case}: no sub-step kernel recorded"
    assert all(n.startswith(family + "<") for n in subs), (case, sorted(subs))


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
            if x0_output_dict is not None:      # the custom-sampler nodes' denoised_output
                x0_output_dict["x0"] = x0
        return callback
    return prepare_callback


# ---------------------------------------------------------------------------------------------------------------
# the node path: LanPaint_KSampler.sample
# ---------------------------------------------------------------------------------------------------------------
NODE = dict(shape=(8, 4, 128, 128), mask="rand", mode="Image First", steps=20, n=5, cfg=5.0, sampler="euler",
            scheduler="karras", model_type="EPS", shift=1.0, wan22=False, opts=None, calls=2,
            modes=None, packed=(True, True), denoise=1.0, window=None, add_noise=True, lam=5.0, step_size=0.2)
# packed: the operands the (first, last) call's sub-steps read.  The fused Euler loop (GraphedJob) and the
# whole-sampler graph (SamplerGraphJob) build the packed known-operand layout once per job; the per-sigma path
# (the engine behind k-diffusion's own loop, and the eager job a SamplerGraphJob records) reads the dense operands.
# window: (start_at_step, end_at_step, return_with_leftover_noise) -- the case calls LanPaint_KSamplerAdvanced, with
# add_noise, lam and step_size as its widgets; otherwise LanPaint_KSampler with `denoise`.
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
    # a step window that returns its leftover noise: the fused loop's last boundary steps to sigma > 0, no
    # max_denoise, the inner-step ramp over a truncated schedule, lambda and step size from the widgets
    "adv-window-leftover": dict(NODE, window=(3, 15, True), lam=8.0, step_size=0.15, calls=4),
    "adv-window-leftover-r128": dict(NODE, shape=(128, 4, 128, 128), window=(3, 15, True), lam=8.0, step_size=0.15,
                                     calls=3),
    # add_noise = disable: a fresh noise image from the generator at every outer step, before that step's Langevin
    # draws -- k-diffusion's loop around the per-sigma graphs, dense operands
    "adv-noise-disabled": dict(NODE, window=(2, 10000, False), add_noise=False, mode="Prompt First", calls=4,
                               modes=[None] * 4, packed=(False, False)),
    "denoise-0.6": dict(NODE, denoise=0.6, calls=4),
    # the sampler draws its own noise between wrapper calls: per-sigma graphs, never a whole-loop graph
    "euler-ancestral": dict(NODE, sampler="euler_ancestral", calls=4, modes=[None] * 4, packed=(False, False)),
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
    window = {}
    if c["window"] is not None:
        start, end, leftover = c["window"]
        window = dict(start_step=start, last_step=end, force_full_denoise=not leftover)
    sig = J.ksampler_sigmas(patcher, c["steps"], c["sampler"], c["scheduler"], c["denoise"], **window)
    md = J.max_denoise(base.model_sampling, sig[0])
    cfg_big = 1.0 if c["model_type"] == "FLUX" else (c["cfg"] if c["mode"] == "Image First" else -0.5)
    hp = O.Hyper(n_steps=c["n"], lam=c["lam"], step_size=c["step_size"], min_step_frac=1.0, flow=flow)
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
        latent = {"samples": y, "noise_mask": mask}

        def call():
            torch.cuda.manual_seed(900 + k)     # the generator state a node without a noise image starts from
            if c["window"] is None:
                (out,) = N.LanPaint_KSampler().sample(patcher, seed, c["steps"], c["cfg"], c["sampler"],
                                                      c["scheduler"], POS, NEG, latent, c["denoise"], c["n"],
                                                      c["mode"], "", N.IMAGE_MODE)
            else:
                (out,) = N.LanPaint_KSamplerAdvanced().sample(
                    patcher, "enable" if c["add_noise"] else "disable", seed, c["steps"], c["cfg"], c["sampler"],
                    c["scheduler"], POS, NEG, latent, start, end, "enable" if leftover else "disable", c["n"],
                    c["lam"], c["step_size"], c["mode"], "", N.IMAGE_MODE)
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

        torch.cuda.manual_seed(900 + k)
        if c["add_noise"]:
            noise = minicomfy.prepare_noise(y, seed)  # ComfyUI's CPU noise image; re-seeds every generator like the node
        else:
            noise = torch.zeros(shape)
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


def _patcher(net, dev, model_type="EPS", shift=1.0, channels=4, opts=None):
    base = minicomfy.BaseModel(net, model_type=getattr(minicomfy.ModelType, model_type), latent_channels=channels,
                               shift=shift)
    patcher = minicomfy.ModelPatcher(base, dev)
    if opts is not None:
        patcher.model_options["lanpaint_b200"] = dict(opts)
    return base, patcher


def test_custom_advanced_flux_job_matches_fp64(cuda_device, monkeypatch):
    """LanPaint_SamplerCustomAdvanced (a GUIDER and a NOISE object) on a Flux latent, simple schedule: both outputs,
    `output` and `denoised_output` (the last step's denoised latent), against the fp64 job."""
    minicomfy.install()
    from lanpaint_b200 import comfy_nodes as N
    N._ENGINES.clear()
    dev, case, shape = cuda_device, "custom-adv-flux", (1, 16, 128, 128)
    base, patcher = _patcher(mixing_denoiser, dev, "FLUX", 1.15, shape[1], {"deferred_max_ms": 1e9})
    store = []
    monkeypatch.setattr(sys.modules["latent_preview"], "prepare_callback", _recorder(store))
    sig = minicomfy.KSampler(patcher, 20, dev, "euler", "simple").sigmas
    hp = O.Hyper(n_steps=5, lam=6.0, step_size=0.25, min_step_frac=1.0, flow=True)
    g = torch.Generator().manual_seed(31)
    y, mask = torch.randn(shape, generator=g), _mask("rand", shape, g)
    gen = _generator(dev)
    modes = []
    for k in range(4):
        if k == 3:
            y, mask = torch.randn(shape, generator=g), _mask("rand", shape, g)
        noise = torch.randn(shape, generator=g)
        store.clear()
        guider = minicomfy.CFGGuider(patcher)
        guider.set_conds(POS, NEG)
        guider.set_cfg(3.5)

        def call():
            torch.cuda.manual_seed(700 + k)
            out, den = N.LanPaint_SamplerCustomAdvanced().sample(
                FixedNoise(50 + k, noise), guider, minicomfy.ksampler("euler"), sig,
                {"samples": y, "noise_mask": mask}, 5, 6.0, 0.25, "Prompt First", "")
            return out["samples"], den["samples"]
        if k in (0, 3):
            (got, got_den), kernels = _sub_kernels(call)
            _assert_torch_tma(f"{case} call {k}", kernels, True)
        else:
            got, got_den = call()
        modes.append(N.LAST_RUN["mode"])
        torch.cuda.synchronize()
        offset = gen.get_offset()
        got_steps = list(store)
        torch.cuda.manual_seed(700 + k)
        want_steps = []
        model = J.Guider(mixing_denoiser, O.FlowSampling(), 3.5, 1.0)       # Flux: cfg_BIG = 1
        dm = _full(mask, shape).to(dev, torch.float64)
        want = J.job(J.SAMPLERS["euler"], model, y.to(dev, torch.float64), noise.to(dev, torch.float64), dm, sig, hp,
                     max_denoise=J.max_denoise(base.model_sampling, sig[0]), callback=lambda i, d: want_steps.append(d))
        assert gen.get_offset() == offset, f"{case} call {k}: generator offset differs from the reference's"
        _check(case, f"call {k} out", got, want)
        _check(case, f"call {k} denoised_output", got_den, want_steps[-1])
        _check_steps(case, f"call {k}", got_steps, want_steps, y.to(dev), (_full(mask, shape) <= 0.5).to(dev))
    assert modes[0] == "eager" and all(m in ("job", "steps") for m in modes[1:]) and N.LAST_RUN["fused"], modes
    N._ENGINES.clear()


def test_av_pack_job_matches_fp64(cuda_device, monkeypatch):
    """A MiniMax-H3 audio-video flat pack of 4.7 M elements through the patched CFGGuider.outer_sample with
    `latent_shapes`: the per-sigma route with the row split, the audio rows' own schedule and target correction at
    every outer step.  No TMA sub-step kernel runs under a row split."""
    minicomfy.install()
    from lanpaint_b200 import comfy_nodes as N
    N._ENGINES.clear()
    monkeypatch.setattr(N, "time_shift_sigma", av_shift_sigma)
    monkeypatch.setattr(N, "time_shift_slope", av_shift_slope)
    dev, case = cuda_device, "av-pack-4.7M"
    n_video, n_audio, sv, sa = 245760, 49152, 3.0, 1.5
    shape = (1, 16, n_video + n_audio)

    def net(x, sigma, cond):
        return mixing_denoiser(x, sigma, cond)
    net.sigma_shift_video, net.sigma_shift_audio = sv, sa
    base, patcher = _patcher(net, dev, "FLOW", 3.0, shape[1])
    N._set_hyper(patcher, num_steps=5, cfg=3.5, prompt_mode="Image First")
    sig = minicomfy.KSampler(patcher, 12, dev, "euler", "simple").sigmas
    hp = O.Hyper(n_steps=5, min_step_frac=1.0, flow=True)
    g = torch.Generator().manual_seed(17)
    gen = _generator(dev)
    for k in range(4):
        if k in (0, 3):
            y = torch.randn(shape, generator=g)
            mask = (torch.rand(shape, generator=g) < 0.5).float()
        noise = torch.randn(shape, generator=g)
        guider = minicomfy.CFGGuider(patcher)
        guider.set_conds(POS, NEG)
        guider.set_cfg(3.5)

        def call():
            torch.cuda.manual_seed(800 + k)
            with N.override_sample_function():
                return type(guider).outer_sample(guider, noise, y, minicomfy.ksampler("euler"), sig, denoise_mask=mask,
                                                 seed=2, latent_shapes=[(1, n_video), (1, n_audio)])
        if k in (0, 3):
            got, kernels = _lp_kernels(call)
            _assert_family(f"{case} call {k}", kernels, "substep_torchvec_kernel")
            assert not any("tma" in n for n in kernels), (case, sorted(kernels))
        else:
            got = call()
        assert N.LAST_RUN["fused"] is False and N.LAST_RUN["mode"] is None, N.LAST_RUN
        torch.cuda.synchronize()
        offset = gen.get_offset()
        torch.cuda.manual_seed(800 + k)
        model = J.Guider(mixing_denoiser, O.FlowSampling(), 3.5, 3.5)
        want = J.job(J.SAMPLERS["euler"], model, y.to(dev, torch.float64), noise.to(dev, torch.float64),
                     mask.to(dev, torch.float64), sig, hp, max_denoise=J.max_denoise(base.model_sampling, sig[0]),
                     audio=J.av_audio(n_video, sv, sa))
        assert gen.get_offset() == offset, f"{case} call {k}: generator offset differs from the reference's"
        _check(case, f"call {k} out", got, want)
    N._ENGINES.clear()


# ---------------------------------------------------------------------------------------------------------------
# inner early stop: the GPU's stop points replayed by the fp64 job, every check restated in fp64
# ---------------------------------------------------------------------------------------------------------------
ES_THRESHOLD = 0.7   # chosen once for the fixed seeds below: 3 outer steps of each job stop mid-loop, and every
ES_MARGIN = 0.01     # distance lands >= 8 % from its threshold in an fp32 CPU run of the same jobs (other draws)


def _ring(known):
    """Free sites with a known 4-neighbour, over the last two axes."""
    near = torch.zeros_like(known)
    near[..., 1:, :] |= known[..., :-1, :]
    near[..., :-1, :] |= known[..., 1:, :]
    near[..., :, 1:] |= known[..., :, :-1]
    near[..., :, :-1] |= known[..., :, 1:]
    return (~known) & near


def _stop_checks(rec, free, ring, threshold_eff, patience_eff):
    """The stopper of one outer step restated in fp64 over the fp64 job's states: lp_stop_stats_f32's two sums
    (free elements, ring elements) of squared differences -- of the VP states around sub-step 0 for the first check,
    of consecutive x0 estimates after that, and of the x0 estimate and its anchor for the drift guard -- each divided
    by its element count as earlystop.py does; then the patience counter.  Returns one dict per check."""
    w_in, w_ring = float(free.sum()), float(ring.sum())

    def stats(a, b):
        d2 = (a - b) ** 2
        return float((d2 * free).sum()) / (w_in + 1e-12), float((d2 * ring).sum()) / (w_ring + 1e-12)
    out, anchor, counter = [], None, 0
    for j, x0 in enumerate(rec["x0"]):
        if j == 0:
            d_in, d_ring = stats(rec["x"][1], rec["x"][0])[0], None
            dist = d_in
        else:
            d_in, d_ring = stats(x0, rec["x0"][j - 1])
            dist = max(d_in, d_ring)
        tested, d_drift = [dist], None
        if dist <= threshold_eff:
            if anchor is None:
                anchor = x0
            else:
                d_drift = max(stats(x0, anchor))
                dist = max(dist, d_drift)
                tested.append(dist)
        else:
            anchor = None
        if dist <= threshold_eff:
            counter += 1
        else:
            counter, anchor = 0, None
        out.append(dict(dist_inpaint=d_in, dist_ring=d_ring, dist_drift=d_drift, dist=dist, patience_counter=counter,
                        stopped=counter >= patience_eff, tested=tested))
    return out


def test_early_stop_job_matches_fp64(cuda_device, monkeypatch):
    """LanPaint_KSampler with the semantic stop on: the un-fused sub-step loop (x0 side output, lp_advance_f32,
    lp_stop_stats_f32, a decision after every sub-step).  The fp64 job stops where the GPU run's trace stopped; every
    recorded distance must equal its fp64 restatement, every decision must be the one the fp64 distances give, and
    every distance must clear the threshold by a margin, so that no decision rests on round-off."""
    minicomfy.install()
    from lanpaint_b200 import comfy_nodes as N
    N._ENGINES.clear()
    dev, case, shape, n = cuda_device, "early-stop", (8, 4, 128, 128), 10
    base, patcher = _patcher(mixing_denoiser, dev)
    trace = []
    patcher.model_options["lanpaint_semantic_stop"] = {"threshold": ES_THRESHOLD, "patience": 1}
    patcher.model_options["lanpaint_semantic_trace"] = trace
    store = []
    monkeypatch.setattr(sys.modules["latent_preview"], "prepare_callback", _recorder(store))
    sig = J.ksampler_sigmas(patcher, 20, "euler", "karras")
    hp = O.Hyper(n_steps=n, min_step_frac=1.0)
    g = torch.Generator().manual_seed(57)
    gen = _generator(dev)
    for k in range(2):
        mid_loop = 0
        y, mask = torch.randn(shape, generator=g), _mask("rand", shape, g)
        seed = 60 + k
        store.clear()
        trace.clear()

        def call():
            (out,) = N.LanPaint_KSampler().sample(patcher, seed, 20, 5.0, "euler", "karras", POS, NEG,
                                                  {"samples": y, "noise_mask": mask}, 1.0, n, "Image First", "",
                                                  N.IMAGE_MODE)
            return out["samples"]
        got, kernels = _lp_kernels(call)
        _assert_family(f"{case} call {k}", kernels, "substep_torchvec_kernel")
        assert any(n_.startswith("advance_") for n_ in kernels) and any(n_.startswith("stop_stats") for n_ in kernels)
        assert N.LAST_RUN["fused"] is False and N.LAST_RUN["mode"] is None, N.LAST_RUN
        torch.cuda.synchronize()
        offset = gen.get_offset()
        got_steps = list(store)
        # the GPU's checks, one group per outer step that ran sub-steps
        groups = []
        for t in trace:
            if t["inner_step"] == 1:
                groups.append([])
            groups[-1].append(t)
        recs = []

        class Recorder(J.Guider):
            """Keeps the latest network input: sub-step 0's is the VE-space state the first check compares with."""

            def __call__(self, x, sigma, model_options=None, seed=None):
                self.last_x = x
                return super().__call__(x, sigma, model_options, seed)
        model = Recorder(mixing_denoiser, O.VESampling(), 5.0, 5.0)

        def on_substep(call):
            rec = {"x": [], "x0": []}
            s = float(sig[call])             # Euler: one wrapper call per outer step

            def hook(i, x_t, state):
                if i == 0:
                    rec["group"] = groups[len(recs)]
                    recs.append(rec)
                    rec["x"].append(model.last_x / (1.0 + s * s) ** 0.5)   # x_t = x / sqrt(1 + VE^2)
                rec["x"].append(x_t)
                rec["x0"].append(state.x0)
                return i + 1 == len(rec["group"]) and rec["group"][-1]["stopped"]
            return hook
        noise = minicomfy.prepare_noise(y, seed)
        want_steps = []
        dm = _full(mask, shape).to(dev, torch.float64)
        want = J.job(J.SAMPLERS["euler"], model, y.to(dev, torch.float64), noise.to(dev, torch.float64), dm, sig, hp,
                     max_denoise=J.max_denoise(base.model_sampling, sig[0]), callback=lambda i, d: want_steps.append(d),
                     on_substep=on_substep)
        assert len(recs) == len(groups), (len(recs), len(groups))
        assert gen.get_offset() == offset, f"{case} call {k}: generator offset differs from the reference's"
        _check(case, f"call {k} out", got, want)
        _check_steps(case, f"call {k}", got_steps, want_steps, y.to(dev), (_full(mask, shape) <= 0.5).to(dev))

        known = (mask.to(dev) <= 0.5).expand(shape)
        free, ring = (~known).double(), _ring(mask.to(dev) <= 0.5).expand(shape).double()
        for s_i, rec in enumerate(recs):
            grp = rec["group"]
            assert len(rec["x0"]) == len(grp)
            abt = float(grp[0]["abt"])
            assert abs(grp[0]["threshold_eff"] - ES_THRESHOLD * min(1.0, 4 * abt * (1 - abt))) <= 1e-6 * ES_THRESHOLD
            want_checks = _stop_checks(rec, free, ring, grp[0]["threshold_eff"], grp[0]["patience_eff"])
            for t, w in zip(grp, want_checks):
                where = f"{case} call {k} outer step {s_i} check {t['inner_step']}"
                for key in ("dist_inpaint", "dist_ring", "dist_drift", "dist"):
                    if w[key] is None:
                        assert t[key] is None, (where, key, t[key])
                    else:
                        assert abs(t[key] - w[key]) <= 1e-4 * abs(w[key]), (where, key, t[key], w[key])
                assert (t["patience_counter"], t["stopped"]) == (w["patience_counter"], w["stopped"]), (where, t, w)
                for d in w["tested"]:
                    assert abs(d / t["threshold_eff"] - 1.0) >= ES_MARGIN, (where, "decision within the margin", d)
            s32 = sig[s_i:s_i + 1].float()
            if grp[-1]["stopped"] and len(grp) < O.inner_steps_for(s32, sig.float(), O.times_from_sigma(s32, False).abt, n):
                mid_loop += 1
        assert mid_loop >= 2, f"{case} call {k}: only {mid_loop} outer steps stopped mid-loop"
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
