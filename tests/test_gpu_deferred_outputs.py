"""What a deferred fused job keeps of each outer step's denoised latent (GraphedJob.run's observe setting).

(a) Through LanPaint_KSampler.sample on minicomfy, at R = 8 and R = 128, for euler and dpmpp_2m (whose previous
    denoised latent a later launch reads): ComfyUI's stock callback without a previewer runs the job as "final", with
    ComfyUI's latent-to-RGB previewer as "preview", and the option deferred_outputs = "full" as today.  The samples are
    bit-identical across the three, the callback runs once per step, x0_output["x0"] is the whole last-step latent and
    the previewer sees, step by step, the bits of the "full" run's x0[:1].  A callback of the user's own still gets
    every step's whole denoised latent.
(b) The row-bounded boundary entry points (lp_boundary_*_rows) on guarded operands: `out` holds exactly out_rows
    rows, nothing past them is written, and every other result is bit-identical to the unbounded call's."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

P = C.c_void_p
STEPS = 20


def _node_run(R, sampler, cuda_device, monkeypatch, option=None, previewer=None, callback=None):
    """Two calls of one request (the eager one, then the deferred whole-job graph): the second call's samples, mode,
    observe setting, x0_output dict and what the stock callback's previewer / a user callback saw."""
    import minicomfy
    from _node_cases import NEG, POS, denoiser
    minicomfy.install()
    from lanpaint_b200 import comfy_nodes as N
    shape = (R, 4, 64, 64)
    g = torch.Generator().manual_seed(R)
    latent = {"samples": torch.randn(shape, generator=g),
              "noise_mask": (torch.rand((R, 1) + shape[2:], generator=g) < 0.5).float()}
    N._ENGINES.clear()
    base = minicomfy.BaseModel(denoiser, model_type=minicomfy.ModelType.EPS, latent_channels=shape[1])
    patcher = minicomfy.ModelPatcher(base, cuda_device)
    patcher.model_options["lanpaint_b200"] = dict({"deferred_max_ms": 1e9}, **(option or {}))
    store = {}
    monkeypatch.setitem(minicomfy.PREVIEW, "previewer", previewer)
    # the stock closure, with an x0_output dict as the custom-sampler nodes pass one
    monkeypatch.setattr(minicomfy.prepare_callback, "__defaults__", (store,))
    if callback is not None:
        monkeypatch.setattr(minicomfy.sys.modules["latent_preview"], "prepare_callback", callback)
    for k in range(2):
        if previewer is not None:
            previewer.seen = []
        calls0 = minicomfy.PROGRESS["calls"]
        torch.cuda.manual_seed(50)
        (out,) = N.LanPaint_KSampler().sample(patcher, 7, STEPS, 5.0, sampler, "karras", POS, NEG, latent, 1.0, 3,
                                              "Image First", "", N.IMAGE_MODE)
    torch.cuda.synchronize()
    job = N.LAST_RUN["job"]
    observe = [k for k, v in job._outs.items() if v is job.outs]
    res = dict(samples=out["samples"].clone(), mode=N.LAST_RUN["mode"], observe=observe,
               x0=store.get("x0"), calls=minicomfy.PROGRESS["calls"] - calls0,
               seen=list(previewer.seen) if previewer is not None else None)
    N._ENGINES.clear()
    return res


@pytest.mark.parametrize("sampler", ["euler", "dpmpp_2m"])
@pytest.mark.parametrize("R", [8, 128])
def test_stock_callback_reads_the_same_under_every_setting(R, sampler, cuda_device, monkeypatch):
    import minicomfy
    full = _node_run(R, sampler, cuda_device, monkeypatch, option={"deferred_outputs": "full"},
                     previewer=minicomfy.Latent2RGBPreviewer())
    final = _node_run(R, sampler, cuda_device, monkeypatch)
    preview = _node_run(R, sampler, cuda_device, monkeypatch, previewer=minicomfy.Latent2RGBPreviewer())
    for name, r in (("full", full), ("final", final), ("preview", preview)):
        assert r["mode"] == "job" and r["observe"] == [name], (name, r["mode"], r["observe"])
        assert r["calls"] == STEPS, (name, r["calls"])
        assert torch.isfinite(r["samples"]).all() and torch.equal(r["samples"], full["samples"]), name
        assert r["x0"].shape[0] == R, name
    # the last step's whole latent, in its own buffer: the "final" / "preview" jobs wrote the "full" job's bits
    assert torch.equal(final["x0"], full["x0"]) and torch.equal(preview["x0"], full["x0"])
    assert len(full["seen"]) == len(preview["seen"]) == STEPS
    for i, (a, b) in enumerate(zip(full["seen"], preview["seen"])):
        assert a.shape[0] == 1 and torch.equal(a, b), i


@pytest.mark.parametrize("R", [8, 128])
def test_a_user_callback_gets_every_whole_latent(R, cuda_device, monkeypatch):
    import minicomfy
    full = _node_run(R, "euler", cuda_device, monkeypatch, option={"deferred_outputs": "full"},
                     previewer=minicomfy.Latent2RGBPreviewer())
    got = []

    def prepare(model, steps, x0_output_dict=None):
        def callback(step, x0, x, total_steps):
            got.append((step, x0.clone()))
        return callback

    user = _node_run(R, "euler", cuda_device, monkeypatch, callback=prepare)
    assert user["observe"] == ["full"] and torch.equal(user["samples"], full["samples"])
    mine = got[-STEPS:]
    assert [s for s, _ in mine] == list(range(STEPS))
    for (step, x0), seen in zip(mine, full["seen"]):
        assert x0.shape[0] == R and torch.equal(x0[:1], seen), step
    assert torch.equal(mine[-1][1], full["x0"])


def test_deferred_outputs_setting_from_the_callback():
    import minicomfy
    minicomfy.install()
    from lanpaint_b200 import comfy_nodes as N
    lp = minicomfy.sys.modules["latent_preview"]
    assert N._deferred_outputs(lp.prepare_callback(None, 4), {}) == "final"
    assert N._deferred_outputs(lp.prepare_callback(None, 4, {}), {"deferred_outputs": "full"}) == "full"
    saved = minicomfy.PREVIEW["previewer"]
    try:
        minicomfy.PREVIEW["previewer"] = minicomfy.Latent2RGBPreviewer()
        assert N._deferred_outputs(lp.prepare_callback(None, 4), {}) == "preview"

        class Animated:      # a previewer that is not ComfyUI's may read every request
            def decode_latent_to_preview_image(self, fmt, x0):
                return None
        minicomfy.PREVIEW["previewer"] = Animated()
        assert N._deferred_outputs(lp.prepare_callback(None, 4), {}) == "full"
    finally:
        minicomfy.PREVIEW["previewer"] = saved
    assert N._deferred_outputs(lambda i, x0, x, n: None, {}) == "full"
    with pytest.raises(ValueError):
        N._deferred_outputs(lp.prepare_callback(None, 4), {"deferred_outputs": "preview"})


# ---- (b) the row bound on guarded operands ---------------------------------------------------------------------
BIG = (5, 4, 120, 136)   # 326400 elements: the TMA-staged torch-stream ancestral kernel
CASES = {
    "known-v4": dict(kernel="known", shape=BIG),
    "known-scalar": dict(kernel="known", shape=(3, 3, 33, 35)),
    "ancestral-torch-tma": dict(kernel="ancestral", shape=BIG),
    "ancestral-philox": dict(kernel="ancestral", shape=(3, 4, 64, 64), philox=True),
    "midpoint": dict(kernel="midpoint", shape=BIG),
    "deis": dict(kernel="deis", shape=BIG),
    "gradient-estimation": dict(kernel="ge", shape=BIG),
}


def _call(lib, c, bounded, rows, hd, y, nz, pm, kn, x, x2, out, d_out, tab, dims, st):
    from lanpaint_b200 import _native
    r = _native.Rng()
    r.mode = _native.RNG_PHILOX if c.get("philox") else _native.RNG_TORCH
    r.seed, r.draw0 = 99, 4096
    ex = (rows,) if bounded else ()
    suffix = "_rows" if bounded else ""
    common = (C.byref(hd), P(y.data_ptr()), P(nz.data_ptr()), P(pm.data.data_ptr()), C.byref(kn.struct))
    tail = (P(tab.data_ptr()), C.byref(dims), st)
    k = c["kernel"]
    if k == "known":
        return getattr(lib, "lp_boundary_known" + suffix)(*common, P(x.data_ptr()), P(out.data_ptr()), *ex,
                                                         C.c_float(-0.2), *tail)
    if k == "ancestral":
        return getattr(lib, "lp_boundary_ancestral" + suffix)(*common, P(x.data_ptr()), P(out.data_ptr()), *ex,
                                                             C.byref(_native.Ancestral(2.0, -0.3, 1.0, 0.5)),
                                                             C.byref(r), *tail)
    if k == "midpoint":
        return getattr(lib, "lp_boundary_midpoint" + suffix)(*common, P(x.data_ptr()), P(x.data_ptr()),
                                                            P(x2.data_ptr()), P(out.data_ptr()), *ex,
                                                            C.byref(_native.Midpoint(2.0, -0.3)), *tail)
    if k == "deis":
        return getattr(lib, "lp_boundary_deis" + suffix)(*common, P(x.data_ptr()), P(out.data_ptr()), *ex,
                                                        P(d_out.data_ptr()), None, None,
                                                        C.byref(_native.Deis(2.0, -0.3, 0.0, 0.0)), *tail)
    return getattr(lib, "lp_boundary_gradient_estimation" + suffix)(
        *common, P(x.data_ptr()), P(out.data_ptr()), *ex, P(d_out.data_ptr()), None,
        C.byref(_native.GradientEstimation(2.0, -0.3, 1.0, 0)), *tail)


@pytest.mark.parametrize("out_rows", [0, 1, 2])
@pytest.mark.parametrize("case", list(CASES))
def test_out_rows_bound_writes_only_its_rows(case, out_rows, cuda_device):
    from lanpaint_b200 import _native
    from lanpaint_b200.engine import pack_known, pack_mask
    from lanpaint_b200.schedule import Hyper, build_table, times_from_sigma
    from _guard import Arena
    c = CASES[case]
    dev, shape = cuda_device, c["shape"]
    R = shape[0]
    per_row, spatial = shape[1] * shape[2] * shape[3], shape[2] * shape[3]
    g = torch.Generator().manual_seed(5)
    y, nz, x0, a = (torch.randn(shape, generator=g).to(dev) for _ in range(4))
    pm = pack_mask((torch.rand((R, 1) + shape[2:], generator=g) < 0.5).to(dev), y)
    dims = _native.Dims(R, per_row, spatial, pm.row_stride, pm.channel_stride)
    kn = pack_known(pm, dims, y, nz)
    s = torch.linspace(0.5, 3.0, R)
    ve, abt, _ = times_from_sigma(s, False)
    tab = torch.from_numpy(build_table(abt.numpy(), ve.numpy(), Hyper(0.2, 5.0, 1.0, 1.0, False))).to(dev)
    hd = _native.Heads(a.data_ptr(), a.data_ptr(), _native.DTYPE_F32, 0, 1.0, 1.0)
    lib = _native.load()
    st = P(torch.cuda.current_stream().cuda_stream)
    # the unbounded call on plain operands
    x, x2, out, d_out = x0.clone(), torch.zeros_like(x0), torch.empty_like(x0), torch.empty_like(x0)
    _native.check(_call(lib, c, False, None, hd, y, nz, pm, kn, x, x2, out, d_out, tab, dims, st), case)
    # the bounded call: `out` placed between guard bands with room for out_rows rows only
    arena = Arena(dev)
    xb = arena.place(x0, name="x")
    x2b = arena.place(torch.zeros_like(x0), name="x2")
    d_outb = arena.place(torch.empty_like(x0), name="d_out")
    outb = arena.place(torch.empty((max(out_rows, 1),) + shape[1:], device=dev), name="out")
    arena.snapshot()
    torch.cuda.synchronize()
    _native.check(_call(lib, c, True, out_rows, hd, y, nz, pm, kn, xb, x2b, outb, d_outb, tab, dims, st), case)
    torch.cuda.synchronize()
    written = {"known": ("x",), "ancestral": ("x",), "midpoint": ("x2",)}.get(c["kernel"], ("x", "d_out"))
    arena.check(case, written=written + (("out",) if out_rows else ()))
    assert torch.equal(xb, x) and torch.equal(x2b, x2), case
    if c["kernel"] in ("deis", "ge"):
        assert torch.equal(d_outb, d_out), case
    if out_rows:
        assert torch.equal(outb, out[:out_rows]), case
