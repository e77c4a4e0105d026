"""GPU: the fused euler_ancestral loop -- lp_boundary_ancestral per launch against fp64, its draw against
torch.randn_like, and whole jobs (node path with the option "fused_ancestral", runner.GraphedJob) against the fp64
job of tests/_job_ref.py and, bit for bit, against the un-fused route."""
import ctypes as C
import sys
import time

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

import _job_ref as J
import _launch_ref as R
import minicomfy
from _node_cases import NEG, POS, mixing_denoiser
from oracle import langevin_oracle as O

pytestmark = pytest.mark.gpu

K = 8            # |got - want| <= K * 2^-24 * magnitude per element, as tests/test_gpu_launch_ref.py
JOB_B = 4e-6     # max|got - want| / max|want| of a whole job, as tests/test_gpu_job_ref.py
P = C.c_void_p
DTYPES = {torch.float32: "float", torch.bfloat16: "__nv_bfloat16", torch.float16: "__half"}
LP_DT = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}
TMA_MIN = 1 << 18


def _native():
    from lanpaint_b200 import _native as n
    return n


def _lib():
    return _native().load()


def _stream():
    return P(torch.cuda.current_stream().cuda_stream)


def _generator(dev):
    torch.cuda.init()
    return torch.cuda.default_generators[dev.index]


def _torch_T(n):
    g, inc = C.c_int64(0), C.c_uint64(0)
    assert _lib().lp_torch_randn_geometry(n, torch.cuda.current_device(), C.byref(g), C.byref(inc)) == 0
    return int(g.value) * 256, int(inc.value)


def _launched(fn):
    """Run fn() (library calls, returning a status) under torch.profiler -> canonical lp:: kernel names."""
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        time.sleep(0.005)
        rc = fn()
        torch.cuda.synchronize()
        time.sleep(0.005)
    assert rc == 0, rc
    return {R.canon(e.name()) for e in prof.profiler.kineto_results.events() if "lp::" in e.name()}


# ---------------------------------------------------------------------------------------------------------------
# 1. one launch against fp64
# ---------------------------------------------------------------------------------------------------------------
def ref_ancestral(a, b, y, noise, known, x, step, xi, next_tab, cfg):
    """lp_boundary_ancestral of the header in fp64 -> dict(out, x) of (value, magnitude) pairs (see _launch_ref)."""
    def expr(m, a, b, y, noise, x, xi):
        A = m.abs
        d = b + m.sub(a, b) * A(cfg) if cfg is not None else a
        out = torch.where(known, y, d)
        x = x + m.sub(x, out) / step.sigma * A(step.down)
        if xi is not None:
            x = x + xi * A(step.s_noise) * A(step.sigma_up)
        if next_tab is not None:
            rn, ry = A(R._row(next_tab, R.T_REPN, x.ndim)), A(R._row(next_tab, R.T_REPY, x.ndim))
            x = torch.where(known, rn * noise + ry * y, x)
        return out, x
    z = torch.zeros((), dtype=torch.float64, device=y.device)
    ops = [R._d(a), z if b is None else R._d(b), R._d(y), R._d(noise), R._d(x), R._d(xi)]
    val = expr(R._Val, *ops)
    mag = expr(R._Mag, *[None if o is None else o.abs() for o in ops])
    return {"out": (val[0], mag[0]), "x": (val[1], mag[1])}


def expect_kernel(c, total, sp):
    H, cb, nx, pk = DTYPES[c["dtype"]], int(c["combine"]), int(c["next"]), int(c["packed"])
    v4 = sp % 4 == 0
    if c["rng"] == "torch":
        T, _ = _torch_T(total)
        calls = -(-total // (4 * T))
        if c.get("tma", 1) and v4 and sp % 16 == 0 and total >= TMA_MIN and T % 1024 == 0 and sp >= 64:
            return f"boundary_ancestral_torch_tma_kernel<{H},{cb},{nx},{pk}>"
        return f"boundary_ancestral_kernel<{4 if v4 and calls <= 65535 else 1},{H},{pk},2>"
    return f"boundary_ancestral_kernel<{4 if v4 else 1},{H},{pk},{ {'tape': 0, 'philox': 1, 'none': -1}[c['rng']] }>"


def table_rows(n_rows, dev, seed):
    """A next-step table: only rep_noise / rep_y are read."""
    g = torch.Generator().manual_seed(seed)
    tab = torch.zeros(n_rows, 32)
    tab[:, R.T_REPN] = torch.rand(n_rows, generator=g) * 3 + 0.05
    tab[:, R.T_REPY] = torch.rand(n_rows, generator=g) * 0.5 + 0.5
    return tab.to(dev)


def run_launch(c, dev, eps_bm=5e-4):
    """-> (x, out, kernels) of one lp_boundary_ancestral call of case c, after checking it against fp64."""
    nat, lib = _native(), _lib()
    shape = c["shape"]
    total, sp = int(np.prod(shape)), int(np.prod(shape[2:]))
    gen = torch.Generator(device=dev).manual_seed(c["seed"])
    bshape = (shape[0], 1) + tuple(shape[2:])
    kind = c.get("mask", "rand")
    known1 = {"rand": lambda: torch.rand(bshape, device=dev, generator=gen) < 0.5,
              "known": lambda: torch.ones(bshape, dtype=torch.bool, device=dev),
              "free": lambda: torch.zeros(bshape, dtype=torch.bool, device=dev)}[kind]()
    m8, known = known1.to(torch.uint8).contiguous(), known1.expand(shape)
    dims = nat.Dims(shape[0], total // shape[0], sp, sp, 0, 0)
    x = torch.randn(shape, device=dev, generator=gen) * 3
    y = torch.randn(shape, device=dev, generator=gen)
    noise = torch.randn(shape, device=dev, generator=gen)
    a = (torch.randn(shape, device=dev, generator=gen) * 1.5).to(c["dtype"])
    b = (a.float() + 0.3 * torch.randn(shape, device=dev, generator=gen)).to(c["dtype"]) if c["combine"] else None
    cfg = 4.5 if c["combine"] else None
    next_tab = table_rows(shape[0], dev, c["seed"]) if c["next"] else None
    out = torch.full(shape, float("nan"), device=dev) if c["out"] else None
    step = nat.Ancestral(1.7, -0.4375 * 1.1, 0.9, 0.0 if c.get("eta0") else 0.6)
    # the draw
    r, xi, slack, keep = nat.Rng(), None, 0.0, []
    seed = c["seed"] * 7919 + 3
    if c["rng"] == "tape":
        xi = torch.randn(shape, device=dev, generator=gen)
        r.mode, r.tape0 = nat.RNG_TAPE, xi.data_ptr()
    elif c["rng"] == "philox":
        xi = torch.from_numpy(R.philox_normals(total, seed, 11 + 5)).to(dev).view(shape)
        st = torch.tensor([seed, 11], dtype=torch.int64, device=dev)     # {seed, base} read from the device
        keep.append(st)
        r.mode, r.seed, r.draw0, r.state = nat.RNG_PHILOX, 0, 5, st.data_ptr()
        slack = eps_bm * abs(step.s_noise * step.sigma_up)
    elif c["rng"] == "torch":
        base = 4 * 37
        g = torch.Generator(device=dev).manual_seed(seed)
        g.set_offset(base)
        xi = torch.randn(shape, device=dev, generator=g)
        st = torch.tensor([seed, base], dtype=torch.int64, device=dev)
        keep.append(st)
        r.mode, r.seed, r.draw0, r.state = nat.RNG_TORCH, 0, 0, st.data_ptr()
    kn = None
    if c["packed"]:
        words = torch.zeros(int(lib.lp_known_words(total)), dtype=torch.int32, device=dev)
        yk, nk = torch.zeros(total + 4, device=dev), torch.zeros(total + 4, device=dev)
        assert lib.lp_pack_known(P(m8.data_ptr()), C.byref(dims), P(y.data_ptr()), P(noise.data_ptr()),
                                 P(words.data_ptr()), P(yk.data_ptr()), P(nk.data_ptr()), _stream()) == 0
        kn = nat.Known(words.data_ptr(), yk.data_ptr(), nk.data_ptr())
        keep += [words, yk, nk]
    hd = nat.Heads(a.data_ptr(), b.data_ptr() if b is not None else None, LP_DT[c["dtype"]], 1 if c["combine"] else 0,
                   cfg or 0.0, cfg or 0.0)
    want = ref_ancestral(a, b, y, noise, known, x, step, xi, next_tab, cfg)
    xg = x.clone()

    def call():
        return lib.lp_boundary_ancestral(C.byref(hd), P(y.data_ptr()), P(noise.data_ptr()), P(m8.data_ptr()),
                                         C.byref(kn) if kn is not None else None, P(xg.data_ptr()),
                                         P(out.data_ptr()) if out is not None else None, C.byref(step),
                                         C.byref(r) if c["rng"] != "none" else None,
                                         P(next_tab.data_ptr()) if next_tab is not None else None, C.byref(dims),
                                         _stream())
    lib.lp_set_option(b"tma", c.get("tma", 1))
    try:
        kernels = _launched(call)
        for _ in range(2):      # CUPTI can, rarely, deliver no record of a kernel that ran: launch again, same inputs
            if kernels:
                break
            xg.copy_(x)
            kernels = _launched(call)
    finally:
        lib.lp_set_option(b"tma", 1)
    label = str(c)
    worst, bad = R.within(xg, want["x"], K, slack)
    assert bad is None, f"{label}: x element {bad}, worst ratio {worst:.3g} > K = {K}"
    if out is not None:
        worst, bad = R.within(out, want["out"], K)
        assert bad is None, f"{label}: out element {bad}, worst ratio {worst:.3g}"
        assert torch.equal(out[known], y[known])
    if c["next"] and c["rng"] != "philox":     # the replace step rounds as lp_prologue_f32 does
        xp = torch.zeros_like(xg)
        assert lib.lp_prologue_f32(P(xp.data_ptr()), P(y.data_ptr()), P(noise.data_ptr()), P(m8.data_ptr()),
                                   P(xp.data_ptr()), None, P(next_tab.data_ptr()), C.byref(dims), _stream()) == 0
        assert torch.equal(xg[known], xp[known])
    assert kernels == {expect_kernel(c, total, sp)}, (label, kernels, expect_kernel(c, total, sp))
    return xg, out, kernels


BASE = dict(shape=(8, 4, 128, 128), dtype=torch.float32, combine=False, next=True, out=True, packed=True, rng="torch",
            seed=1)
F32, BF16, F16 = torch.float32, torch.bfloat16, torch.float16
LAUNCHES = {
    # the TMA kernel: dtypes, combine, next, out, packed / dense
    "tma-f32-cfg-next-packed": dict(BASE, combine=True),
    "tma-f32-cfg-last-dense": dict(BASE, combine=True, next=False, packed=False, seed=2),
    "tma-bf16-next-dense-noout": dict(BASE, dtype=BF16, packed=False, out=False, seed=3),
    "tma-f16-last-packed": dict(BASE, dtype=F16, next=False, seed=4),
    "tma-f32-eta0": dict(BASE, eta0=True, seed=5),
    "tma-all-known": dict(BASE, mask="known", seed=6),
    "tma-all-free": dict(BASE, mask="free", dtype=BF16, seed=7),
    "tma-all-known-dense-last": dict(BASE, mask="known", packed=False, next=False, seed=8),
    "tma-r128-tail-first": dict(BASE, shape=(128, 4, 128, 128), combine=True, seed=9),
    "tma-r128-dense-bf16": dict(BASE, shape=(128, 4, 128, 128), dtype=BF16, packed=False, out=False, seed=10),
    "tma-wan-partial-groups": dict(BASE, shape=(1, 16, 21, 80, 45), seed=11),
    "tma-wan-dense-f16": dict(BASE, shape=(1, 16, 21, 80, 45), dtype=F16, packed=False, seed=12),
    "tma-min": dict(BASE, shape=(1, 4, 256, 256), seed=13),
    # the LDG kernel: torch vec4 / scalar, philox, tape, no draw
    "ldg-torch-small": dict(BASE, shape=(1, 4, 32, 32), seed=20),
    "ldg-torch-small-dense-cfg": dict(BASE, shape=(1, 4, 32, 32), packed=False, combine=True, seed=21),
    "ldg-torch-ragged": dict(BASE, shape=(1, 3, 7, 9), seed=22),
    "ldg-torch-ragged-dense-f16": dict(BASE, shape=(2, 3, 7, 9), packed=False, dtype=F16, next=False, seed=23),
    "ldg-torch-below-tma-min": dict(BASE, shape=(3, 4, 128, 128), dtype=BF16, seed=24),
    "ldg-philox-big": dict(BASE, rng="philox", seed=25),
    "ldg-philox-ragged-dense": dict(BASE, rng="philox", shape=(1, 3, 7, 9), packed=False, seed=26),
    "ldg-tape-big-cfg": dict(BASE, rng="tape", combine=True, seed=27),
    "ldg-tape-small-dense-bf16": dict(BASE, rng="tape", shape=(1, 4, 32, 32), packed=False, dtype=BF16, seed=28),
    "ldg-tape-ragged": dict(BASE, rng="tape", shape=(1, 3, 7, 9), next=False, seed=29),
    "ldg-none-big-last": dict(BASE, rng="none", next=False, eta0=True, seed=30),
    "ldg-none-r128-dense": dict(BASE, rng="none", shape=(128, 4, 128, 128), packed=False, eta0=True, seed=31),
    "ldg-none-ragged": dict(BASE, rng="none", shape=(1, 3, 7, 9), eta0=True, out=False, seed=32),
    "ldg-philox-eta0": dict(BASE, rng="philox", shape=(1, 4, 32, 32), eta0=True, seed=33),
}


@pytest.mark.parametrize("case", list(LAUNCHES))
def test_launch_matches_fp64(case, cuda_device):
    c = LAUNCHES[case]
    x, out, kernels = run_launch(c, cuda_device)
    if case.startswith("tma-"):
        assert all(k.startswith("boundary_ancestral_torch_tma_kernel<") for k in kernels), kernels
        x2, out2, k2 = run_launch(dict(c, tma=0), cuda_device)     # the LDG kernel on the same inputs: same bits
        assert all(k.startswith("boundary_ancestral_kernel<4,") for k in k2), k2
        assert torch.equal(x, x2) and (out is None or torch.equal(out, out2))


# ---------------------------------------------------------------------------------------------------------------
# 2. the draw is torch.randn_like's
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(8, 4, 128, 128), (1, 16, 21, 80, 45), (1, 4, 32, 32), (1, 3, 7, 9)])
def test_the_draw_is_torch_randn_like(shape, cuda_device):
    """x = head = 0 on an all-free mask with s_noise = sigma_up = 1 leaves x = xi: it equals torch.randn_like at the
    generator's offset bit for bit, on the TMA kernel and on both LDG mappings."""
    nat, lib, dev = _native(), _lib(), cuda_device
    total, sp = int(np.prod(shape)), int(np.prod(shape[2:]))
    gen = _generator(dev)
    torch.cuda.manual_seed(4242)
    torch.randn(1000, device=dev)             # somewhere inside the stream
    seed, off = gen.initial_seed(), gen.get_offset()
    assert off > 0
    x = torch.zeros(shape, device=dev)
    want = torch.randn_like(x)
    assert gen.get_offset() - off == _torch_T(total)[1]
    zero, m8 = torch.zeros(shape, device=dev), torch.zeros((shape[0], 1) + tuple(shape[2:]), dtype=torch.uint8, device=dev)
    dims = nat.Dims(shape[0], total // shape[0], sp, sp, 0, 0)
    hd = nat.Heads(zero.data_ptr(), None, 0, 0, 0.0, 0.0)
    step = nat.Ancestral(2.0, -0.5, 1.0, 1.0)
    r = nat.Rng(mode=nat.RNG_TORCH, seed=seed, draw0=off)
    for tma in (1, 0):
        x.zero_()
        lib.lp_set_option(b"tma", tma)
        try:
            rc = lib.lp_boundary_ancestral(C.byref(hd), P(zero.data_ptr()), None, P(m8.data_ptr()), None, P(x.data_ptr()),
                                           None, C.byref(step), C.byref(r), None, C.byref(dims), _stream())
        finally:
            lib.lp_set_option(b"tma", 1)
        assert rc == 0
        assert torch.equal(x, want), (shape, tma)


# ---------------------------------------------------------------------------------------------------------------
# 3. whole jobs through the nodes
# ---------------------------------------------------------------------------------------------------------------
def _rel(got, want):
    got = got.to(device=want.device, dtype=torch.float64)
    return float((got - want).abs().max() / want.abs().max())


def _recorder(store):
    def prepare_callback(model, steps, x0_output_dict=None):
        def callback(step, x0, x, total_steps):
            store.append((step, x0.detach().clone()))
        return callback
    return prepare_callback


def _sub_kernels(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    names = {R.canon(e.name()) for e in prof.profiler.kineto_results.events() if "lp::" in e.name()}
    return out, names


NODE = dict(shape=(8, 4, 128, 128), steps=20, n=5, cfg=5.0, window=None, calls=4, deferred=True, eta=None)
NODE_CASES = {
    "b8-deferred": dict(NODE),
    "b8-steps": dict(NODE, deferred=False),
    "b8-window-leftover": dict(NODE, window=(3, 15, True)),
    "b8-window-leftover-steps": dict(NODE, window=(3, 15, True), deferred=False),
    "r128": dict(NODE, shape=(128, 4, 128, 128), calls=3),
    "r128-window-leftover": dict(NODE, shape=(128, 4, 128, 128), window=(3, 15, True), calls=3, deferred=False),
}


def _node_call(N, patcher, c, latent, seed, k):
    torch.cuda.manual_seed(900 + k)
    if c["window"] is None:
        (out,) = N.LanPaint_KSampler().sample(patcher, seed, c["steps"], c["cfg"], "euler_ancestral", "karras", POS, NEG,
                                              latent, 1.0, c["n"], "Image First", "", N.IMAGE_MODE)
    else:
        start, end, leftover = c["window"]
        (out,) = N.LanPaint_KSamplerAdvanced().sample(
            patcher, "enable", seed, c["steps"], c["cfg"], "euler_ancestral", "karras", POS, NEG, latent, start, end,
            "enable" if leftover else "disable", c["n"], 5.0, 0.2, "Image First", "", N.IMAGE_MODE)
    return out["samples"]


@pytest.mark.parametrize("case", list(NODE_CASES))
def test_node_job_matches_fp64_and_the_unfused_route(case, cuda_device, monkeypatch):
    """eager -> capture -> replay -> (a new seed and mask on the same graphs): every call within JOB_B of the fp64
    job, per-step denoised latents equal y at known positions, generator offset the reference's, and the result and
    every step's denoised latent bit-identical to the same call with the option off (the per-sigma route)."""
    c = NODE_CASES[case]
    minicomfy.install()
    from lanpaint_b200 import comfy_nodes as N
    N._ENGINES.clear()
    dev, shape = cuda_device, c["shape"]
    base = minicomfy.BaseModel(mixing_denoiser, model_type=minicomfy.ModelType.EPS, latent_channels=shape[1], shift=1.0)
    fused = minicomfy.ModelPatcher(base, dev)
    fused.model_options["lanpaint_b200"] = {"fused_ancestral": True, "deferred_callbacks": c["deferred"],
                                            "deferred_max_ms": 1e9}
    plain = minicomfy.ModelPatcher(base, dev)
    store = []
    monkeypatch.setattr(sys.modules["latent_preview"], "prepare_callback", _recorder(store))
    window = {}
    if c["window"] is not None:
        window = dict(start_step=c["window"][0], last_step=c["window"][1], force_full_denoise=not c["window"][2])
    sig = J.ksampler_sigmas(fused, c["steps"], "euler_ancestral", "karras", 1.0, **window)
    if c["window"] is not None:
        assert float(sig[-1]) > 0
    md = J.max_denoise(base.model_sampling, sig[0])
    hp = O.Hyper(n_steps=c["n"], lam=5.0, step_size=0.2, min_step_frac=1.0, flow=False)
    g = torch.Generator().manual_seed(sum(map(ord, case)))
    y = torch.randn(shape, generator=g)
    mask = (torch.rand((shape[0], 1) + shape[2:], generator=g) < 0.5).float()
    gen = _generator(dev)
    modes = []
    for k in range(c["calls"]):
        seed = 40 + k // 3
        if k == 3:
            y = torch.randn(shape, generator=g)
            mask = (torch.rand((shape[0], 1) + shape[2:], generator=g) < 0.5).float()
        latent = {"samples": y, "noise_mask": mask}
        store.clear()
        if k in (0, c["calls"] - 1):    # which kernels the eager job and the last replayed job ran
            got, kernels = _sub_kernels(lambda: _node_call(N, fused, c, latent, seed, k))
            subs = {n for n in kernels if n.startswith("substep")}
            assert subs and all(n.startswith("substep_torch_tma_kernel<") and n.endswith(",1>") for n in subs), subs
            bnd = {n for n in kernels if n.startswith("boundary")}
            # every step with a draw ran the packed TMA kernel (a window's last step without a next replace step); a
            # last step to sigma 0 the LDG kernel without a draw
            last = {"boundary_ancestral_kernel<4,float,1,-1>"} if c["window"] is None else set()
            assert bnd - last and all(n.startswith("boundary_ancestral_torch_tma_kernel<float,") and n.endswith(",1>")
                                      for n in bnd - last), bnd
        else:
            got = _node_call(N, fused, c, latent, seed, k)
        modes.append(N.LAST_RUN["mode"])
        assert N.LAST_RUN["fused"] and N.LAST_RUN["job"].sampler == "euler_ancestral"
        torch.cuda.synchronize()
        offset, got_steps = gen.get_offset(), list(store)

        # the un-fused route: option off
        store.clear()
        ref = _node_call(N, plain, c, latent, seed, k)
        assert N.LAST_RUN["mode"] is None and not N.LAST_RUN["fused"]
        torch.cuda.synchronize()
        assert gen.get_offset() == offset
        assert torch.equal(got, ref), f"{case} call {k}: fused and un-fused results differ, max {float((got - ref).abs().max())}"
        assert len(store) == len(got_steps) == len(sig) - 1
        for (i, d), (j, e) in zip(got_steps, store):
            assert i == j and torch.equal(d, e), f"{case} call {k}: denoised[{i}] differs from the un-fused route's"

        # fp64
        torch.cuda.manual_seed(900 + k)
        noise = minicomfy.prepare_noise(y, seed)
        yd = y.to(dev, torch.float64)
        dm = minicomfy.repeat_to_batch_size(mask, shape[0]).expand(shape).to(dev, torch.float64)
        want_steps = []
        model = J.Guider(mixing_denoiser, O.VESampling(), c["cfg"], c["cfg"])
        want = J.job(J.SAMPLERS["euler_ancestral"], model, yd, noise.to(dev, torch.float64), dm, sig, hp,
                     max_denoise=md, callback=lambda i, d: want_steps.append(d))
        assert gen.get_offset() == offset, f"{case} call {k}: generator offset differs from the reference's"
        assert _rel(got, want) <= JOB_B, (case, k, _rel(got, want))
        known = (dm <= 0.5)
        for (i, d), w in zip(got_steps, want_steps):
            assert _rel(d, w) <= JOB_B, (case, k, i, _rel(d, w))
            assert torch.equal(d[known], y.to(dev)[known])
    assert modes == ["eager"] + ["job" if c["deferred"] else "steps"] * (c["calls"] - 1), modes
    N._ENGINES.clear()


def test_eta_and_s_noise_reach_the_fused_loop(cuda_device):
    """A SAMPLER object with extra_options eta / s_noise through LanPaint_SamplerCustom: the fused job equals the
    per-sigma route bit for bit, eta = 0 included (the draw is still consumed: same generator offset)."""
    minicomfy.install()
    from lanpaint_b200 import comfy_nodes as N
    N._ENGINES.clear()
    dev, shape = cuda_device, (2, 4, 64, 64)
    base = minicomfy.BaseModel(mixing_denoiser, model_type=minicomfy.ModelType.EPS, latent_channels=4, shift=1.0)
    g = torch.Generator().manual_seed(77)
    latent = {"samples": torch.randn(shape, generator=g),
              "noise_mask": (torch.rand((2, 1, 64, 64), generator=g) < 0.5).float()}
    gen = _generator(dev)
    for eta, s_noise in ((0.0, 1.0), (0.5, 1.1)):
        res = []
        for on in (True, False, True):
            patcher = minicomfy.ModelPatcher(base, dev)
            patcher.model_options["lanpaint_b200"] = {"fused_ancestral": on}
            sig = minicomfy.KSampler(patcher, 8, dev, "euler_ancestral", "karras").sigmas
            sampler = minicomfy.ksampler("euler_ancestral", {"eta": eta, "s_noise": s_noise})
            torch.cuda.manual_seed(5)
            out, _ = N.LanPaint_SamplerCustom().sample(patcher, sampler, sig, True, 3, 4.0, POS, NEG, latent, 3,
                                                       "Image First")
            assert N.LAST_RUN["fused"] == on and N.LAST_RUN["mode"] == ("eager" if on else None)
            if on:
                step = N.LAST_RUN["job"].ancestral[0][0]
                assert step.s_noise == C.c_float(s_noise).value and (step.sigma_up == 0.0) == (eta == 0.0)
            res.append((out["samples"].clone(), gen.get_offset()))
        assert torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][0], res[2][0]), (eta, s_noise)
        assert res[0][1] == res[1][1] == res[2][1]
    N._ENGINES.clear()


# ---------------------------------------------------------------------------------------------------------------
# runner.GraphedJob directly
# ---------------------------------------------------------------------------------------------------------------
def _engine(rng, merge=True):
    from lanpaint_b200.engine import LanPaint
    from lanpaint_b200.runner import SynthDenoiser, VESampling
    return LanPaint(SynthDenoiser(VESampling()), NSteps=4, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2,
                    MinStepFrac=1.0, rng=rng, batched_replace="per_sample", merge_noise=merge)


@pytest.mark.parametrize("shape", [(2, 4, 64, 64), (8, 4, 128, 128)])
@pytest.mark.parametrize("sigmas", ["to-zero", "leftover"])
def test_graphed_job_equals_the_unfused_definition(shape, sigmas, cuda_device):
    """eager / per-step graphs / whole-job graph, fused and un-fused, each bit-equal to euler_ancestral_inpaint, with
    the generator left where the definition leaves it.  Per-step graphs are also replayed out of capture order: a
    step's draws are addressed from the job's {seed, base} block, not from whatever was captured first."""
    from lanpaint_b200.runner import GraphedJob, HostSchedule, euler_ancestral_inpaint, karras_sigmas
    dev = cuda_device
    ks = karras_sigmas(8)
    sched = HostSchedule(ks if sigmas == "to-zero" else ks[1:-2], shape[0], 4)
    g = torch.Generator().manual_seed(9)
    y, noise = torch.randn(shape, generator=g).to(dev), torch.randn(shape, generator=g).to(dev)
    mask = (torch.rand((shape[0], 1) + shape[2:], generator=g) < 0.5).float().to(dev)
    gen = _generator(dev)
    for eta, s_noise in ((1.0, 1.0), (0.0, 1.0), (0.6, 0.9)):
        torch.cuda.manual_seed(31)
        want = euler_ancestral_inpaint(_engine("torch"), y, noise, mask, sched, eta=eta, s_noise=s_noise)
        offset = gen.get_offset()
        for fused in (True, False):
            job = GraphedJob(_engine("torch"), sched, shape, dev, fused_euler=fused, sampler="euler_ancestral", eta=eta,
                             s_noise=s_noise)
            n = len(sched.steps)
            assert job.draws == sum(2 * st.n_inner - 1 for st in sched.steps if st.n_inner > 0) + (
                n if sigmas == "leftover" else n - 1)
            for mode in ("eager", "steps", "job", "steps"):
                torch.cuda.manual_seed(31)
                got = job.run(y, noise, mask, mode=mode)
                assert gen.get_offset() == offset, (fused, mode)
                assert torch.equal(got, want), (eta, s_noise, fused, mode, float((got - want).abs().max()))
        if eta == 1.0:    # per-step graphs captured last step first
            job = GraphedJob(_engine("torch"), sched, shape, dev, sampler="euler_ancestral")
            job.load_inputs(y, noise, mask)
            for i in reversed(range(n)):
                job._graph_for(("step", i, False), lambda p, i=i: job._step(i, p, False), True)
            torch.cuda.manual_seed(31)
            assert torch.equal(job.run(y, noise, mask, mode="steps"), want)


def test_philox_job_matches_fp64_fed_the_same_draws(cuda_device):
    """rng = "philox" (un-merged kicks): the fused job against the fp64 job whose every draw -- Langevin and the
    sampler's -- is lp_fill_normal_f32 at the next draw index of the same stream."""
    from lanpaint_b200.runner import GraphedJob, HostSchedule, karras_sigmas
    nat, lib, dev = _native(), _lib(), cuda_device
    shape, n_inner = (8, 4, 128, 128), 4
    ks = karras_sigmas(8)
    sched = HostSchedule(ks, shape[0], n_inner)
    g = torch.Generator().manual_seed(19)
    y, noise = torch.randn(shape, generator=g).to(dev), torch.randn(shape, generator=g).to(dev)
    mask = (torch.rand((shape[0], 1) + shape[2:], generator=g) < 0.5).float().to(dev)
    gen = _generator(dev)
    torch.cuda.manual_seed(123)
    seed, off = gen.initial_seed(), gen.get_offset()
    job = GraphedJob(_engine("philox", merge=False), sched, shape, dev, sampler="euler_ancestral", eta=0.8, s_noise=1.0)
    got = job.run(y, noise, mask, mode="eager")
    assert gen.get_offset() == off + 4 * job.draws
    count = [0]

    def draw(like):
        xi = torch.empty(like.shape, device=dev)
        r = nat.Rng(mode=nat.RNG_PHILOX, seed=seed, draw0=off // 4 + count[0])
        assert lib.lp_fill_normal_f32(P(xi.data_ptr()), xi.numel(), C.byref(r), _stream()) == 0
        count[0] += 1
        return xi.to(like.dtype)

    coef = job.engine.inner_model.coef

    class Net:      # SynthDenoiser in the job's dtype
        def __init__(self):
            self.inner_model, self.model_sampling = self, O.VESampling()

        def __call__(self, x, sigma, model_options=None, seed=None):
            return coef[0] * x + coef[1] * torch.tanh(x) + coef[2], coef[3] * x + coef[4]

    def sampler(model, x, sigmas, callback=None, draw=None):
        from unittest import mock
        with mock.patch.object(torch, "randn_like", lambda like, **kw: draw(like)):
            return minicomfy.sample_euler_ancestral(model, x, sigmas, callback=callback, eta=0.8, s_noise=1.0)
    hp = O.Hyper(n_steps=n_inner, lam=5.0, step_size=0.2, min_step_frac=1.0, flow=False)
    dm = (1.0 - mask).expand(shape).to(torch.float64)
    want = J.job(sampler, Net(), y.double(), noise.double(), dm, torch.tensor(ks), hp, draw=draw)
    assert count[0] == job.draws
    assert _rel(got, want) <= 2e-5, _rel(got, want)      # the synthetic network's fp32 tanh on top of JOB_B


# ---------------------------------------------------------------------------------------------------------------
# 5. routing
# ---------------------------------------------------------------------------------------------------------------
def test_routing_and_cache_separation(cuda_device):
    """Option absent: the per-sigma route as before.  Option on: fused only for euler_ancestral on a plain inpainting
    job (not with an inner early stop, not with a zero noise image, not for another sampler).  Toggling the option,
    or switching between euler and euler_ancestral on one schedule, never reuses the other's job."""
    minicomfy.install()
    from lanpaint_b200 import comfy_nodes as N
    N._ENGINES.clear()
    dev, shape = cuda_device, (2, 4, 64, 64)
    base = minicomfy.BaseModel(mixing_denoiser, model_type=minicomfy.ModelType.EPS, latent_channels=4, shift=1.0)
    g = torch.Generator().manual_seed(3)
    latent = {"samples": torch.randn(shape, generator=g), "noise_mask": (torch.rand((2, 1, 64, 64), generator=g) < 0.5).float()}

    def run(patcher, sampler="euler_ancestral", **kw):
        torch.cuda.manual_seed(1)
        (out,) = N.LanPaint_KSampler().sample(patcher, 5, 8, 4.0, sampler, "karras", POS, NEG, latent, 1.0, 3,
                                              "Image First", "", N.IMAGE_MODE, **kw)
        return out["samples"], N.LAST_RUN["mode"], N.LAST_RUN["fused"], N.LAST_RUN["job"]

    patcher = minicomfy.ModelPatcher(base, dev)
    seen = []
    for on in (None, True, None, True, False, True):      # one patcher, the option toggled between calls
        if on is None:
            patcher.model_options.pop("lanpaint_b200", None)
        else:
            patcher.model_options["lanpaint_b200"] = {"fused_ancestral": on}
        out, mode, fused, job = run(patcher)
        seen.append((out, mode, fused, job))
        assert fused == bool(on) and (mode is None) == (not on)
    assert [m for _, m, _, _ in seen] == [None, "eager", None, "job", None, "job"]
    assert all(torch.equal(seen[0][0], o) for o, _, _, _ in seen[1:])
    assert seen[1][3] is seen[3][3] is seen[5][3] and seen[1][3].sampler == "euler_ancestral"
    # euler on the same schedule and options: its own job, then back
    out_e, mode_e, fused_e, job_e = run(patcher, "euler")
    assert fused_e and job_e is not seen[1][3] and job_e.sampler == "euler" and mode_e == "eager"
    out_a, mode_a, _, job_a = run(patcher)
    assert job_a is seen[1][3] and torch.equal(out_a, seen[0][0]) and not torch.equal(out_e, out_a)
    _, _, _, job_e2 = run(patcher, "euler")
    assert job_e2 is job_e
    # another sampler with the option on: not the fused loop
    _, mode_h, fused_h, _ = run(patcher, "heun")
    assert not fused_h
    N._ENGINES.clear()


def test_zero_noise_and_early_stop_are_not_fused(cuda_device):
    minicomfy.install()
    from lanpaint_b200 import comfy_nodes as N
    from lanpaint_b200.engine import LanPaint
    N._ENGINES.clear()
    dev, shape = cuda_device, (2, 4, 64, 64)
    base = minicomfy.BaseModel(mixing_denoiser, model_type=minicomfy.ModelType.EPS, latent_channels=4, shift=1.0)
    patcher = minicomfy.ModelPatcher(base, dev)
    patcher.model_options["lanpaint_b200"] = {"fused_ancestral": True}
    g = torch.Generator().manual_seed(3)
    latent = {"samples": torch.randn(shape, generator=g), "noise_mask": (torch.rand((2, 1, 64, 64), generator=g) < 0.5).float()}
    # add_noise = disable: a zero noise image, regenerated at every outer step by the per-sigma route
    torch.cuda.manual_seed(1)
    N.LanPaint_KSamplerAdvanced().sample(patcher, "disable", 5, 8, 4.0, "euler_ancestral", "karras", POS, NEG, latent, 0,
                                         10000, "disable", 3, 5.0, 0.2, "Image First", "", N.IMAGE_MODE)
    assert N.LAST_RUN["mode"] is None and not N.LAST_RUN["fused"]
    # the gate itself, on an engine with an inner early-stop threshold / an AV pack / a tape
    class K:    # what _fused_ancestral_ok reads of the wrapper
        audio_indicator = None
        sigmas_host = [3.0, 1.0, 0.0]
    ks = minicomfy.ksampler("euler_ancestral")
    eng = LanPaint(None, NSteps=3, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2, rng="torch")
    dm = torch.ones(1)
    ok = lambda k=K, e=eng, mo={}, s=ks: N.KSAMPLER._fused_ancestral_ok(s, k, dm, mo, e)   # noqa: E731
    assert ok()
    assert not N.KSAMPLER._fused_ancestral_ok(ks, K, None, {}, eng)
    av = type("AV", (K,), {"audio_indicator": torch.ones(1)})
    assert not ok(k=av)
    assert not ok(mo={"denoise_mask_function": lambda *a, **k: None})
    assert not ok(mo={"lanpaint_semantic_stop": {}})
    assert not ok(e=LanPaint(None, NSteps=3, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2, rng="torch",
                             EarlyStopThreshold=1e-3))
    assert not ok(s=minicomfy.ksampler("euler"))
    assert not ok(k=type("Z", (K,), {"sigmas_host": [3.0, 0.0, 0.0]}))
    N._ENGINES.clear()
