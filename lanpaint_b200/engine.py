"""H100-native (sm_90a) LanPaint engine: the reference's `LanPaint` class seam, fused.

Drop-in for `src/LanPaint/lanpaint.py:7-157` (constructor and `__call__`
signature, in-place rewrite of `x`, returned `out`, `ValueError("Model output
is empty")`), but between two model calls it issues ONE kernel
(`lp_substep_f32`) where the reference issues ~89, and no host sync inside the
sub-step loop.  The model (`self.inner_model`) stays an opaque PyTorch call.

Differences from the reference that a caller can observe, all deliberate:
  * inputs must live on a CUDA device (there is no CPU/eager fallback; a
    missing library or a CPU tensor raises);
  * `latent_mask` is treated as binary (thresholded at 0.5).  The reference's
    own callers always binarise it first (src/LanPaint/nodes.py:281-283);
  * per-sample scalars (sigma, alpha-bar) are read back to the host once per
    outer step to build the coefficient table in fp64 (the reference syncs
    1+N times per outer step: lanpaint.py:51,205);
  * Gaussian draws: `rng="torch"` (default) reproduces the CUDA global
    generator's `randn_like` stream bit for bit, in the reference's draw order,
    and advances the generator identically; `rng="philox"` is a cheaper
    counter-based stream; a `NoiseTape` makes the draws explicit inputs.
"""
from __future__ import annotations

import ctypes as C
import weakref
from typing import List, Optional, Sequence

import numpy as np
import torch

from . import _native
from .schedule import Hyper, build_table, mean_half_dt
from .state import LangevinState

_P = C.c_void_p


class NoiseTape:
    """Explicit Gaussian draws, consumed in the reference's order (SURVEY 8a quirk 6):
    [regeneration draw if noise~0], then 1 draw for sub-step 0 and 2 per later sub-step."""

    def __init__(self, draws: Sequence[torch.Tensor]):
        self.draws = list(draws)
        self.pos = 0

    def next(self, like: torch.Tensor) -> torch.Tensor:
        if self.pos >= len(self.draws):
            raise IndexError("noise tape exhausted")
        t = self.draws[self.pos]
        self.pos += 1
        if t.shape != like.shape:
            raise ValueError(f"tape draw {self.pos - 1} has shape {tuple(t.shape)}, need {tuple(like.shape)}")
        if t.device != like.device or t.dtype != torch.float32 or not t.is_contiguous():
            t = t.to(device=like.device, dtype=torch.float32).contiguous()
        return t


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _stream_ptr(device: torch.device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def _f32c(t: torch.Tensor) -> torch.Tensor:
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


class CfgPair:
    """Raw network outputs of one cond/uncond evaluation plus the two guidance scales.

    The patched guider returns this instead of the two combined tensors when no user hook needs
    them materialised (comfy_nodes.sampling_function_LanPaint); the engine then feeds cond/uncond
    straight to `lp_substep_cfg_f32`, which does both `uncond + (cond - uncond)*scale` combines in
    registers.  `heads()` gives the eager equivalent for any other consumer."""

    __slots__ = ("cond", "uncond", "cfg", "cfg_big")

    def __init__(self, cond: torch.Tensor, uncond: torch.Tensor, cfg: float, cfg_big: float):
        self.cond, self.uncond, self.cfg, self.cfg_big = cond, uncond, float(cfg), float(cfg_big)

    def heads(self):
        d = self.cond - self.uncond
        return self.uncond + d * self.cfg, self.uncond + d * self.cfg_big


class PackedMask:
    """uint8 known-region mask + the strides the kernels index it with.  `known`, when set, is the known-operand
    layout (`KnownOperands`) of this mask and one job's y and noise: the launches of that job then read the packed
    operands where a kernel can (`pack_known`)."""

    def __init__(self, data: torch.Tensor, row_stride: int, channel_stride: int):
        self.data = data
        self.row_stride = row_stride
        self.channel_stride = channel_stride
        self.known = None


class KnownOperands:
    """The known-operand layout of lp_known (include/lanpaint_b200.h): per 32 latent elements one word of known
    bits and one count of the known elements before them, plus y and the noise image at known elements only.
    y and the noise image are read only at known positions and are constant for a job, so a kernel that streams
    them reads 4 B per known element instead of 4 B per element.  Buffers are sized for `total` elements whatever
    the mask, so one set serves every job of a shape (CUDA graphs keep their addresses)."""

    def __init__(self, total: int, device, with_noise: bool = True):
        lib = _native.load()
        n_words = int(lib.lp_known_words(total))
        if n_words < 0:
            raise ValueError(f"{total} elements: too many for the known-operand layout")
        self.total = total
        self.words = torch.empty(n_words, dtype=torch.int32, device=device)
        self.y = torch.empty(total + 4, dtype=torch.float32, device=device)
        self.noise = torch.empty(total + 4, dtype=torch.float32, device=device) if with_noise else None
        self.struct = _native.Known(self.words.data_ptr(), self.y.data_ptr(),
                                    self.noise.data_ptr() if with_noise else None)


def pack_known(pm: PackedMask, dims, y: torch.Tensor, noise: Optional[torch.Tensor] = None,
               out: Optional[KnownOperands] = None) -> KnownOperands:
    """Fill (or allocate) the known-operand layout of mask `pm` and the dense fp32 y / noise (lp_pack_known, three
    small launches on the current stream).  The dense operands stay in use by every kernel that reads them dense."""
    total = y.numel()
    if out is None or out.total != total or (noise is not None and out.noise is None):
        out = KnownOperands(total, y.device, noise is not None)
    lib = _native.load()
    rc = lib.lp_pack_known(_P(pm.data.data_ptr()), C.byref(dims), _P(y.data_ptr()),
                           _P(noise.data_ptr()) if noise is not None else None, _P(out.words.data_ptr()),
                           _P(out.y.data_ptr()), _P(out.noise.data_ptr()) if noise is not None else None,
                           _P(_stream_ptr(y.device)))
    _native.check(rc, "lp_pack_known")
    return out


def pack_mask(latent_mask: torch.Tensor, like: torch.Tensor) -> PackedMask:
    """latent_mask (1 = known) of any shape broadcastable to `like` -> PackedMask.

    A mask that is constant over channels by construction (shape [B,1,...] or an
    expanded view) is stored once per spatial site: 1/C byte per latent element."""
    B, Cc = like.shape[0], like.shape[1]
    spatial = int(np.prod(like.shape[2:])) if like.ndim > 2 else 1
    m = latent_mask
    if m.device != like.device:
        m = m.to(like.device)
    while m.ndim < like.ndim:
        m = m.unsqueeze(0)
    if m.ndim != like.ndim:
        raise ValueError(f"mask rank {m.ndim} does not match latent rank {like.ndim}")
    chan_bcast = m.shape[1] == 1 or (m.shape[1] == Cc and m.stride(1) == 0)
    if chan_bcast and Cc > 1:
        m = m[:, :1]
        target = (B, 1) + tuple(like.shape[2:])
    else:
        target = tuple(like.shape)
    if tuple(m.shape) != target:
        m = m.expand(target)
    lib = _native.load()
    if m.dtype in (torch.uint8, torch.bool):
        data = (m != 0).to(torch.uint8).contiguous()
    else:
        src = _f32c(m)
        data = torch.empty(target, dtype=torch.uint8, device=like.device)
        rc = lib.lp_pack_mask_f32(_P(src.data_ptr()), _P(data.data_ptr()), src.numel(), 0,
                                  _P(_stream_ptr(like.device)))
        _native.check(rc, "lp_pack_mask_f32")
    if target[1] == 1 and Cc > 1:
        return PackedMask(data, spatial, 0)
    return PackedMask(data, Cc * spatial, spatial)


def options_fingerprint(o, depth: int = 0):
    """A cheap structural identity of a model_options-like object: primitives by value, containers two
    levels deep, everything else (tensors, callables, patches) by object identity.  Graph caches key on it
    because a captured graph bakes in whatever the model read from these options at capture time."""
    if isinstance(o, (str, int, float, bool, type(None))):
        return o
    if isinstance(o, dict) and depth < 3:
        return tuple((str(k), options_fingerprint(v, depth + 1)) for k, v in sorted(o.items(), key=lambda kv: str(kv[0])))
    if isinstance(o, (list, tuple)) and depth < 3:
        return tuple(options_fingerprint(v, depth + 1) for v in o)
    if isinstance(o, torch.Tensor) and o.numel() <= 1024:
        # small tensors (ComfyUI's transformer_options["sample_sigmas"], ...) are re-created per job with
        # the same values: identify them by content
        return ("tensor", tuple(o.shape), str(o.dtype), tuple(o.detach().reshape(-1).tolist()))
    return id(o)


def _tensor_key(t: torch.Tensor):
    """What can change under us without the object changing: storage address, layout, in-place writes.
    Inference tensors (ComfyUI runs nodes under torch.inference_mode) have no version counter."""
    try:
        version = t._version
    except RuntimeError:
        version = None
    return (t.data_ptr(), version, tuple(t.shape), tuple(t.stride()), t.dtype)


class _Ident:
    """Identity of a tensor for caching: the SAME Python object (a freed tensor's address is routinely
    handed to a new one by the caching allocator) in the same state."""

    __slots__ = ("ref", "key")

    def __init__(self, t: torch.Tensor):
        self.ref = weakref.ref(t)
        self.key = _tensor_key(t)

    def matches(self, t: torch.Tensor) -> bool:
        return self.ref() is t and self.key == _tensor_key(t)


class _IdentityCache:
    """value cached per tensor identity: avoids recomputing per outer step."""

    def __init__(self):
        self._ident: Optional[_Ident] = None
        self.value = None

    def get(self, t: torch.Tensor):
        if self._ident is not None and self._ident.matches(t):
            return self.value
        return None

    def put(self, t: torch.Tensor, value):
        self._ident = _Ident(t)
        self.value = value


class LanPaint:
    """Same constructor / call surface as the reference engine (lanpaint.py:8,44).

    Extra keyword-only knobs (all also settable per call through
    ``model_options["lanpaint_b200"] = {...}``):
      rng             "torch" | "philox" | NoiseTape
      batched_replace "reference" (lanpaint.py:87-92 literal: flow-form replace whenever
                      sigma has more than one element) | "per_sample" (every sample is an
                      independent B=1 request; uses model_sampling.noise_scaling's form)
      replace_mode    "probe" (derive the linear form of noise_scaling from a 4-point host
                      probe; falls back to "call" if it is not linear) | "call"
      merge_noise     rng="philox" only: a fused launch applies two independent Gaussian kicks with
                      nothing observing the state in between, so it draws one normal with the summed
                      variance (identical chain in distribution, half the RNG work)
      cuda_graph      False | True: capture the whole outer step (model calls included) into one
                      CUDA graph per (shape, sub-step count) and replay it; falls back to eager
                      launches if the model is not capture-safe.  The graph bakes in the model object,
                      whatever it read from model_options (both are part of the cache key) and `seed`
                      (by value; not part of the key), and reads latent_image / noise / mask from static
                      copies refreshed whenever the source tensor changes identity or version
      graph_after     0: capture at first use (one warm-up pass of the step on a side stream first);
                      k > 0: run a configuration eagerly the first k times it is seen and capture it the
                      next time, without a warm-up pass (what the node path uses: no wasted model calls)
    """

    def __init__(self, Model, NSteps, Friction, Lambda, Beta, StepSize, IS_FLUX=False, IS_FLOW=False,
                 EarlyStopThreshold=0.0, EarlyStopPatience=1, EarlyStopHook=None, MinStepFrac=0.0, *,
                 rng="torch", batched_replace="reference", replace_mode="probe", cuda_graph=False,
                 merge_noise=True, graph_after=0):
        self.n_steps = NSteps
        self.chara_lamb = Lambda
        self.IS_FLUX = IS_FLUX
        self.IS_FLOW = IS_FLOW
        self.step_size = StepSize
        self.inner_model = Model
        self.friction = Friction
        self.chara_beta = Beta
        self.min_step_frac = MinStepFrac
        self.img_dim_size = None
        self.early_stop_threshold = EarlyStopThreshold
        self.early_stop_patience = EarlyStopPatience
        self.early_stop_hook = EarlyStopHook
        self.rng = rng
        self.batched_replace = batched_replace
        self.replace_mode = replace_mode
        self.cuda_graph = cuda_graph
        self.merge_noise = merge_noise
        # capture a configuration the (graph_after+1)-th time it is seen; 0 = immediately, with a warm-up pass
        self.graph_after = graph_after
        # part of the graph cache key in place of id(inner_model) when the caller (the node layer) already
        # guarantees that a re-bound inner_model is functionally the one the graphs were captured with
        self.graph_model_token = None
        self._graphs = {}
        self._graph_seen = {}
        self._graph_keep = []
        self._graph_statics = {}
        self.max_live_shapes = 4   # workspaces / static graph buffers kept per (device, shape)
        # statistics a caller (bench, tests) can read back
        self.launches = 0
        self.model_calls = 0
        self.substeps_done = 0
        self._mask_cache = _IdentityCache()
        self._noise_zero_cache = _IdentityCache()
        self._av_cache = _IdentityCache()
        self._av_mask_cache = _IdentityCache()
        self._replace_probe_cache = {"sampling": None, "seen": {}}
        self._ws = {}
        self.stats_reduce = None  # frame_shard.py: sums the early stopper's two statistics over the shards of a latent
        self.kernel_timer = None  # set to a list to collect (flags, start_event, stop_event) per substep launch
        _native.load()  # fail at construction, loudly, if the CUDA library is absent

    def reset_counters(self):
        self.launches = self.model_calls = self.substeps_done = 0

    # ---- small helpers kept for API compatibility (lanpaint.py:23-43) ----------
    def add_none_dims(self, array):
        while array.ndim < self.img_dim_size:
            array = array.unsqueeze(array.ndim)
        return array

    def remove_none_dims(self, array):
        return array[(slice(None),) + (0,) * (self.img_dim_size - 1)]

    def unpack_model_output(self, output):
        if isinstance(output, CfgPair):
            return output.heads()
        if isinstance(output, (tuple, list)):
            if len(output) >= 2:
                return output[0], output[1]
            if len(output) == 1:
                return output[0], output[0]
            raise ValueError("Model output is empty")
        return output, output

    def sigma_x(self, abt):
        return abt ** 0

    def sigma_y(self, abt):
        return self.chara_beta * abt ** 0

    # ---- workspace -------------------------------------------------------------
    def _workspace(self, like: torch.Tensor, rows: int):
        key = (like.device, tuple(like.shape), rows)
        ws = self._ws.get(key)
        if ws is None:
            ws = {
                "c": torch.empty_like(like, dtype=torch.float32, memory_format=torch.contiguous_format),
                "table_dev": torch.empty((rows, _native.TABLE_STRIDE), dtype=torch.float32, device=like.device),
            }
            while len(self._ws) >= self.max_live_shapes:   # a few live shapes (alternating requests), oldest out
                self._ws.pop(next(iter(self._ws)))
            self._ws[key] = ws
        return ws

    # ---- replace-step linear form (lanpaint.py:85-94) ----------------------------
    def _replace_form(self, sigma_host: np.ndarray, scalar_sigma: bool, n_rows: int, mode: str, batched: str):
        """Returns (rep_noise[rows], rep_y[rows]) or None when noise_scaling must be called."""
        sampling = self.inner_model.inner_model.model_sampling
        if not scalar_sigma and batched == "reference":
            ns = float(getattr(sampling, "noise_scale", 1.0))
            s32 = sigma_host.astype(np.float32)
            rep_n = (s32 * np.float32(ns)).astype(np.float64)
            rep_y = (np.float32(1.0) - s32).astype(np.float64)
            return rep_n, rep_y
        if mode != "probe":
            return None
        rn, ry = [], []
        cache = self._replace_probe_cache            # one probe per distinct sigma of one model_sampling object
        if cache.get("sampling") is not sampling or len(cache["seen"]) > 4096:
            cache["sampling"], cache["seen"] = sampling, {}
        seen = cache["seen"]
        for s in (sigma_host if not scalar_sigma else sigma_host[:1]):
            s = float(s)
            form = seen.get(s)
            if form is None:
                form = seen[s] = _probe_noise_scaling(sampling, s) or False
            if form is False:
                return None
            rn.append(form[0])
            ry.append(form[1])
        if scalar_sigma:
            rn, ry = rn * n_rows, ry * n_rows
        return np.asarray(rn, dtype=np.float64), np.asarray(ry, dtype=np.float64)

    # ---- the call ----------------------------------------------------------------
    def __call__(self, x, latent_image, noise, sigma, latent_mask, current_times, model_options, seed,
                 n_steps=None, current_times_audio=None, audio_indicator=None, audio_correction=None):
        self.img_dim_size = len(x.shape)
        self.latent_image = latent_image
        self.noise = noise
        self.audio_indicator = audio_indicator
        self.current_times_audio = current_times_audio
        self.audio_correction = audio_correction
        if not (isinstance(x, torch.Tensor) and x.is_cuda):
            raise RuntimeError("lanpaint_b200.LanPaint needs CUDA tensors: there is no CPU or eager fallback "
                               "(the reference engine is the CPU implementation)")
        if x.numel() == 0:  # an empty batch: nothing to update, nothing to draw, no model call
            return torch.empty_like(x)
        opts = {}
        if isinstance(model_options, dict):
            opts = model_options.get("lanpaint_b200", {}) or {}
        rng = opts.get("rng", self.rng)

        # every launch below goes to the current stream of x's device: make that device current for the call
        # (a process that drives several GPUs -- ComfyUI multi-GPU, thread-per-device replicas -- may not have)
        with torch.cuda.device(x.device):
            # lanpaint.py:51-52 -- add_noise disabled: a fresh noise image every outer step
            if self._noise_is_zero(self.noise):
                self.noise = self._regen_noise(self.noise, rng)
            if n_steps is None:
                n_steps = self.n_steps
            return self.LanPaint(x, sigma, latent_mask, current_times, n_steps, model_options, seed,
                                 self.IS_FLUX, self.IS_FLOW, _opts=opts)

    def _noise_is_zero(self, noise: torch.Tensor) -> bool:
        hit = self._noise_zero_cache.get(noise)
        if hit is None:
            hit = bool(torch.mean(torch.abs(noise)) < 1e-8)  # one sync per distinct noise tensor
            self._noise_zero_cache.put(noise, hit)
        return hit

    def _regen_noise(self, noise: torch.Tensor, rng) -> torch.Tensor:
        if isinstance(rng, NoiseTape):
            return rng.next(noise)
        return torch.randn_like(noise)  # global generator, exactly the reference's draw

    def LanPaint(self, x, sigma, latent_mask, current_times, n_steps, model_options, seed, IS_FLUX, IS_FLOW,
                 _opts=None):
        opts = _opts or {}
        rng = opts.get("rng", self.rng)
        batched = opts.get("batched_replace", self.batched_replace)
        rmode = opts.get("replace_mode", self.replace_mode)
        use_graph = opts.get("cuda_graph", self.cuda_graph)
        dev = x.device
        flow = bool(IS_FLUX or IS_FLOW)
        if self.audio_indicator is not None and self.current_times_audio is not None:
            return self._av_call(x, sigma, latent_mask, current_times, n_steps, model_options, seed, flow, opts)
        input_x = x
        B = x.shape[0]
        per_row = x.numel() // B
        spatial = int(np.prod(x.shape[2:])) if x.ndim > 2 else 1
        VE_Sigma, abt, Flow_t = current_times

        # ---- per-sample scalars on the host: one read-back, or none if the caller already holds
        # sigma / current_times as CPU tensors (the sync-free path bench.py and the graphed runner use)
        def flat(t, where):
            t = t.reshape(-1).to(device=where, dtype=torch.float32)
            return t if t.numel() == B else t.expand(B)
        t_model_src = Flow_t if flow else VE_Sigma
        scal = (sigma, VE_Sigma, abt, t_model_src)
        where = torch.device("cpu") if all(t.device.type == "cpu" for t in scal) else dev
        host = torch.stack([flat(t, where) for t in scal]).cpu().numpy()
        sigma_h, ve_h, abt_h, tm_h = host[0], host[1], host[2], host[3]
        hyper = Hyper(self.step_size, self.chara_lamb, self.chara_beta, self.min_step_frac, flow)

        # ---- operands ----
        y = _f32c(self.latent_image if self.latent_image.device == dev else self.latent_image.to(dev))
        nz = _f32c(self.noise if self.noise.device == dev else self.noise.to(dev))
        pm = self._mask_cache.get(latent_mask) if isinstance(latent_mask, torch.Tensor) else None
        if isinstance(latent_mask, PackedMask):
            pm = latent_mask
        elif pm is None:
            pm = pack_mask(latent_mask, x)
            self._mask_cache.put(latent_mask, pm)
            self.launches += 1
        dims = _native.Dims(B, per_row, spatial, pm.row_stride, pm.channel_stride)
        stopper = self._make_stopper(model_options, pm, x, abt_h, dims)

        scalar_sigma = sigma.numel() == 1
        form = self._replace_form(sigma_h, scalar_sigma, B, rmode, batched)
        if form is None:
            rep_n, rep_y = np.ones(B), np.zeros(B)  # `known` is computed by noise_scaling itself (lanpaint.py:88)
        else:
            rep_n, rep_y = form
        table_np = build_table(abt_h, ve_h, hyper, rep_n, rep_y)

        # lanpaint.py:205: a non-positive mean step skips the dynamics (and its model calls)
        active = n_steps if mean_half_dt(abt_h, hyper) > 0.0 else 0
        plan = _DrawPlan(rng, x, active)

        if use_graph and stopper is None and plan.mode != _native.RNG_TAPE:
            out = self._graphed_step(x, y, nz, pm, dims, table_np, tm_h, sigma_h, sigma.shape, active, plan,
                                     form is None, model_options, seed)
            if out is not None:
                plan.finish()
                self.substeps_done += active
                return out if out.dtype == input_x.dtype else out.to(input_x.dtype)

        xm = x if (x.dtype == torch.float32 and x.is_contiguous()) else _f32c(x)
        ws = self._workspace(xm, B)
        tab = ws["table_dev"]
        tab.copy_(torch.from_numpy(table_np))  # pageable H2D: staged before this returns, no aliasing hazard
        t_model = torch.from_numpy(tm_h).to(dev) if t_model_src.device.type == "cpu" else t_model_src.reshape(-1)
        sigma_dev = sigma.to(dev)
        out = torch.empty_like(xm)
        done = self._launch_sequence(xm, y, nz, pm, dims, tab, t_model, sigma_dev, ws["c"], out, active, plan,
                                     form is None, model_options, seed, stopper, None, current_times=current_times)
        plan.finish()
        self.substeps_done += done
        if xm is not input_x:
            input_x.copy_(xm)
        return out if out.dtype == input_x.dtype else out.to(input_x.dtype)

    # ---- planned calls: everything host-side done ahead, the call itself is capture-safe -------------------
    def plan_item(self, B: int, sigma_host: torch.Tensor, times, n_steps: int, device, sigma_shape=None):
        """Everything `LanPaint()` derives on the host from (sigma, current_times) for ONE wrapper call, as device
        constants: coefficient table, model timestep, sigma.  Used by runner.SamplerGraphJob, which records the
        sigma sequence of a sampler's first (eager) job and then captures the whole sampler loop: the captured
        calls must not read anything back.  Returns None when noise_scaling is not a linear form."""
        flow = bool(self.IS_FLUX or self.IS_FLOW)
        VE_Sigma, abt, Flow_t = times

        def flat(t):
            t = t.reshape(-1).to(device="cpu", dtype=torch.float32)
            return t if t.numel() == B else t.expand(B)
        host = torch.stack([flat(t) for t in (sigma_host, VE_Sigma, abt, Flow_t if flow else VE_Sigma)]).numpy()
        sigma_h, ve_h, abt_h, tm_h = host[0], host[1], host[2], host[3]
        hyper = Hyper(self.step_size, self.chara_lamb, self.chara_beta, self.min_step_frac, flow)
        form = self._replace_form(sigma_h, sigma_host.numel() == 1, B, self.replace_mode, self.batched_replace)
        if form is None:
            return None
        table_np = build_table(abt_h, ve_h, hyper, form[0], form[1])
        active = n_steps if mean_half_dt(abt_h, hyper) > 0.0 else 0
        shape = tuple(sigma_shape) if sigma_shape is not None else tuple(sigma_host.shape)
        return {"table": torch.from_numpy(table_np).to(device), "t_model": torch.from_numpy(tm_h.copy()).to(device),
                "sigma": sigma_host.to(device=device, dtype=torch.float32).reshape(shape), "active": int(active)}

    def run_planned(self, x, item, y, nz, pm, dims, cbuf, plan, rng_state, model_options, seed, discard_heads=False):
        """One wrapper call from a plan_item: no host read-back, no H2D copy, no generator access -- only kernel
        launches and the model calls, i.e. capturable as part of a larger CUDA graph.  x is rewritten in place.
        discard_heads: see `_launch_sequence`."""
        if not (x.is_cuda and x.dtype == torch.float32 and x.is_contiguous()):
            raise RuntimeError("planned LanPaint call needs a contiguous fp32 CUDA state tensor")
        self.img_dim_size = x.ndim
        out = torch.empty_like(x)
        done = self._launch_sequence(x, y, nz, pm, dims, item["table"], item["t_model"], item["sigma"], cbuf, out,
                                     item["active"], plan, False, model_options, seed, None, rng_state,
                                     discard_heads=discard_heads)
        self.substeps_done += done
        return out

    # ---- the launch sequence of one outer step (shared by the eager path and graph capture) ----
    def _launch_sequence(self, xm, y, nz, pm, dims, tab, t_model, sigma_dev, cbuf, out, active, plan, call_scaling,
                         model_options, seed, stopper, rng_state, euler_coef=None, skip_prologue=False,
                         next_table=None, current_times=None, ancestral=None, discard_heads=False, multistep=None,
                         midpoint=None, deis=None, ge=None, heun=None, out_rows=None):
        """discard_heads: the caller owns the network's outputs and nothing reads them once the update kernel that
        consumes them has run (`heads_discardable`), so that kernel may drop them from the L2 unwritten
        (LP_HEADS_DEAD).  Only the fused loop's launches take it; the early-stop loop hands the heads to the stopper.
        multistep: (lp_multistep, the previous step's denoised latent or None): the boundary is
        lp_boundary_multistep, the update of a host-owned sample_dpmpp_2m loop.
        midpoint: (lp_midpoint, x_base, x_out): the boundary is lp_boundary_midpoint, one update of a host-owned
        sample_dpm_2 loop, with xm -- the state this call's sub-steps ran on -- as its x_in.
        deis: (lp_deis, d_out, d_prev1, d_prev2), each buffer or None: the boundary is lp_boundary_deis, the update of a
        host-owned sample_deis loop.
        ge: (lp_gradient_estimation, d_out, d_prev), each buffer or None: the boundary is
        lp_boundary_gradient_estimation, the update of a host-owned sample_gradient_estimation loop.
        heun: (lp_heun, x_base, out_prev): the boundary is lp_boundary_heun, the corrector of a host-owned sample_heun
        loop, with x_base (the state the step started from, updated in place) as its x, xm -- the state this call's
        sub-steps ran on -- as its x2, and out_prev the step's first call's denoised latent.
        out_rows: `out` holds only its first out_rows rows (the boundary's row-bounded form, lp_boundary_*_rows);
        None: every row.  Not for multistep and heun, whose out a later launch reads whole."""
        lib = _native.load()
        dev = xm.device
        stream = _P(_stream_ptr(dev))
        F = _native
        noise_arg = nz
        # the known-operand layout, when the owner of y / nz / pm built it for exactly these operands
        kn = getattr(pm, "known", None)
        if call_scaling:  # opaque noise_scaling: call it like the reference does (lanpaint.py:88)
            sampling = self.inner_model.inner_model.model_sampling
            noise_arg = _f32c(sampling.noise_scaling(self.add_none_dims(sigma_dev), nz, y))
        # prologue: replace step + change of variables (lanpaint.py:85-99); a host-owned Euler loop has
        # already applied it inside the previous step's lp_step_boundary_f32
        if not skip_prologue:
            rc = lib.lp_prologue_f32(_P(xm.data_ptr()), _P(y.data_ptr()), _P(noise_arg.data_ptr()),
                                     _P(pm.data.data_ptr()), _P(xm.data_ptr()), None, _P(tab.data_ptr()),
                                     C.byref(dims), stream)
            _native.check(rc, "lp_prologue_f32")
            self.launches += 1
        done = 0
        for i in range(active):
            first = i == 0
            has_next = i + 1 < active
            self.model_calls += 1
            if stopper is None or first:
                heads = self.inner_model(xm, t_model, model_options=model_options, seed=seed)
                if isinstance(heads, CfgPair) and stopper is None and heads.cond.dtype == torch.float32 \
                        and heads.uncond.dtype == torch.float32:
                    hd, keep = _heads(heads.cond, heads.uncond, xm, True, heads.cfg, heads.cfg_big,
                                      dead=discard_heads)
                else:
                    h0, h1 = self.unpack_model_output(heads)
                    hd, keep = _heads(h0, h1, xm, dead=discard_heads and stopper is None)
            if stopper is None:
                # fused: post-model half of sub-step i + pre-model half of sub-step i+1
                flags = (F.SUBSTEP_FIRST if first else 0) | (F.SUBSTEP_FUSE_NEXT if has_next else 0)
                merge = has_next and plan.mode == F.RNG_PHILOX and self.merge_noise
                if merge:  # one Gaussian with the summed variance instead of two (philox stream only)
                    flags |= F.SUBSTEP_MERGE_NOISE
                r = plan.rng_struct(2 if (has_next and not merge) else 1, rng_state)
                ev = self._event_pair(flags) if self.kernel_timer is not None else None
                # heads of any dtype; with a CfgPair both CFG combines happen inside the kernel
                if kn is not None:
                    rc = lib.lp_substep_known(_P(xm.data_ptr()), C.byref(hd), _P(y.data_ptr()), _P(pm.data.data_ptr()),
                                              C.byref(kn.struct), _P(cbuf.data_ptr()), None, None, _P(tab.data_ptr()),
                                              C.byref(dims), C.byref(r), flags, stream)
                else:
                    rc = lib.lp_substep(_P(xm.data_ptr()), C.byref(hd), _P(y.data_ptr()), _P(pm.data.data_ptr()),
                                        _P(cbuf.data_ptr()), None, None, _P(tab.data_ptr()), C.byref(dims), C.byref(r),
                                        flags, stream)
                if ev is not None:
                    ev[1].record()
                _native.check(rc, "lp_substep")
                self.launches += 1
                done += 1
                continue
            # early-stop loop (lanpaint.py:116-142): the decision to stop after sub-step i must be taken
            # before the first half-advance of sub-step i+1 is applied, so that half is its own launch
            if first and stopper is not None:
                x_before = xm.clone()          # state before sub-step 0 (its check has no previous x0)
                x0e_prev = None
            custom_prev = xm.clone() if stopper.has_custom_distance_fn else None
            if not first:
                r = plan.rng_struct(1, rng_state)
                rc = lib.lp_advance_f32(_P(xm.data_ptr()), _P(cbuf.data_ptr()), _P(pm.data.data_ptr()),
                                        _P(tab.data_ptr()), C.byref(dims), C.byref(r), 1, stream)
                _native.check(rc, "lp_advance_f32")
                self.launches += 1
                heads = self.inner_model(xm, t_model, model_options=model_options, seed=seed)
                h0, h1 = self.unpack_model_output(heads)
                hd, keep = _heads(h0, h1, xm)
            flags = (F.SUBSTEP_FIRST if first else 0) | F.SUBSTEP_STORE_C
            x0e = stopper.next_x0e_buffer(xm)
            r = plan.rng_struct(1, rng_state)
            rc = lib.lp_substep(_P(xm.data_ptr()), C.byref(hd), _P(y.data_ptr()), _P(pm.data.data_ptr()),
                                _P(cbuf.data_ptr()), None, _P(x0e.data_ptr()), _P(tab.data_ptr()), C.byref(dims),
                                C.byref(r), flags, stream)
            _native.check(rc, "lp_substep")
            self.launches += 1
            done += 1
            inv_s = tab[:, _native.T_INVS].reshape((-1,) + (1,) * (xm.ndim - 1))
            # what a user distance_fn may read (lanpaint.py:121-129): the float latent_mask of the latent's
            # shape and the (VE, abt, flow_t) triple -- unpacked only when such a hook exists
            ctx_mask = pm
            if stopper.has_custom_distance_fn:
                if getattr(stopper, "_ctx_mask", None) is None:
                    m = pm.data.reshape(-1).to(torch.float32)
                    stopper._ctx_mask = (m.reshape(xm.shape) if m.numel() == xm.numel()
                                         else pm.data.to(torch.float32).expand(xm.shape))
                ctx_mask = stopper._ctx_mask
            ctx = {"step": i, "steps_done": i + 1, "n_steps": active, "mask": ctx_mask, "latent_image": y,
                   "current_times": current_times, "seed": seed}
            stop = stopper.step(i=i, n_steps=active, x_before=x_before if first else None, x_after=xm,
                                x0_prev=x0e_prev, x0_cur=x0e, table=tab,
                                custom_prev=(lambda: custom_prev * inv_s) if custom_prev is not None else None,
                                custom_cur=(lambda: xm * inv_s) if custom_prev is not None else None, ctx=ctx)
            x0e_prev = x0e
            if stop:
                break

        # final denoise + known-region paste (lanpaint.py:151-157) [+ Euler update + next replace step when the host
        # owns the sampler loop]: one lp_boundary launch, CFG combine folded in when the guider handed raw predictions
        out_heads = self.inner_model(xm, sigma_dev, model_options=model_options, seed=seed)
        self.model_calls += 1
        if isinstance(out_heads, CfgPair) and out_heads.cond.dtype == torch.float32 \
                and out_heads.uncond.dtype == torch.float32:
            hd, keep = _heads(out_heads.cond, out_heads.uncond, xm, True, out_heads.cfg, out_heads.cfg,
                              dead=discard_heads)
        else:
            mo, _ = self.unpack_model_output(out_heads)
            hd, keep = _heads(mo, None, xm, dead=discard_heads)
        rows = () if out_rows is None else (out_rows,)   # the out_rows argument of the row-bounded forms
        if (multistep is not None or heun is not None) and rows:
            raise ValueError("the multistep and heun boundaries store every row of out")
        if ancestral is not None:
            # host-owned sample_euler_ancestral loop: (lp_ancestral, whether the sampler draws at this step).  Its
            # randn_like comes after the step's Langevin draws, so its position is taken here, not earlier
            step, draws = ancestral
            r = plan.rng_struct(1, rng_state) if draws else None
            rc = (lib.lp_boundary_ancestral_rows if rows else lib.lp_boundary_ancestral)(
                C.byref(hd), _P(y.data_ptr()), _P(nz.data_ptr()), _P(pm.data.data_ptr()),
                C.byref(kn.struct) if kn is not None and kn.noise is not None else None,
                _P(xm.data_ptr()), _P(_ptr(out)), *rows, C.byref(step),
                C.byref(r) if r is not None else None, _P(next_table.data_ptr()) if next_table is not None else None,
                C.byref(dims), stream)
            _native.check(rc, "lp_boundary_ancestral")
            self.launches += 1
            return done
        if multistep is not None:
            step, old = multistep
            rc = lib.lp_boundary_multistep(C.byref(hd), _P(y.data_ptr()), _P(nz.data_ptr()), _P(pm.data.data_ptr()),
                                           C.byref(kn.struct) if kn is not None and kn.noise is not None else None,
                                           _P(xm.data_ptr()), _P(_ptr(out)), _P(_ptr(old)), C.byref(step),
                                           _P(next_table.data_ptr()) if next_table is not None else None,
                                           C.byref(dims), stream)
            _native.check(rc, "lp_boundary_multistep")
            self.launches += 1
            return done
        if midpoint is not None:
            step, x_base, x_out = midpoint
            rc = (lib.lp_boundary_midpoint_rows if rows else lib.lp_boundary_midpoint)(
                C.byref(hd), _P(y.data_ptr()), _P(nz.data_ptr()), _P(pm.data.data_ptr()),
                C.byref(kn.struct) if kn is not None and kn.noise is not None else None,
                _P(xm.data_ptr()), _P(x_base.data_ptr()), _P(x_out.data_ptr()), _P(_ptr(out)), *rows,
                C.byref(step), _P(next_table.data_ptr()) if next_table is not None else None, C.byref(dims), stream)
            _native.check(rc, "lp_boundary_midpoint")
            self.launches += 1
            return done
        if deis is not None:
            step, d_out, p1, p2 = deis
            rc = (lib.lp_boundary_deis_rows if rows else lib.lp_boundary_deis)(
                C.byref(hd), _P(y.data_ptr()), _P(nz.data_ptr()), _P(pm.data.data_ptr()),
                C.byref(kn.struct) if kn is not None and kn.noise is not None else None,
                _P(xm.data_ptr()), _P(_ptr(out)), *rows, _P(_ptr(d_out)), _P(_ptr(p1)), _P(_ptr(p2)),
                C.byref(step), _P(next_table.data_ptr()) if next_table is not None else None, C.byref(dims), stream)
            _native.check(rc, "lp_boundary_deis")
            self.launches += 1
            return done
        if ge is not None:
            step, d_out, d_prev = ge
            rc = (lib.lp_boundary_gradient_estimation_rows if rows else lib.lp_boundary_gradient_estimation)(
                C.byref(hd), _P(y.data_ptr()), _P(nz.data_ptr()), _P(pm.data.data_ptr()),
                C.byref(kn.struct) if kn is not None and kn.noise is not None else None, _P(xm.data_ptr()),
                _P(_ptr(out)), *rows, _P(_ptr(d_out)), _P(_ptr(d_prev)), C.byref(step),
                _P(next_table.data_ptr()) if next_table is not None else None, C.byref(dims), stream)
            _native.check(rc, "lp_boundary_gradient_estimation")
            self.launches += 1
            return done
        if heun is not None:
            step, x_base, out_prev = heun
            rc = lib.lp_boundary_heun(C.byref(hd), _P(y.data_ptr()), _P(nz.data_ptr()), _P(pm.data.data_ptr()),
                                      C.byref(kn.struct) if kn is not None and kn.noise is not None else None,
                                      _P(x_base.data_ptr()), _P(xm.data_ptr()), _P(out_prev.data_ptr()), _P(_ptr(out)),
                                      C.byref(step), _P(next_table.data_ptr()) if next_table is not None else None,
                                      C.byref(dims), stream)
            _native.check(rc, "lp_boundary_heun")
            self.launches += 1
            return done
        fused_next = next_table is not None and euler_coef is not None
        if kn is not None and (kn.noise is not None or not fused_next):
            rc = (lib.lp_boundary_known_rows if rows else lib.lp_boundary_known)(
                C.byref(hd), _P(y.data_ptr()), _P(nz.data_ptr()) if fused_next else None, _P(pm.data.data_ptr()),
                C.byref(kn.struct), _P(xm.data_ptr()) if euler_coef is not None else None, _P(_ptr(out)), *rows,
                C.c_float(euler_coef or 0.0), _P(next_table.data_ptr()) if fused_next else None, C.byref(dims), stream)
        elif rows:
            raise ValueError("a row-bounded out needs the known-operand layout")
        else:
            rc = lib.lp_boundary(C.byref(hd), _P(y.data_ptr()), _P(nz.data_ptr()) if fused_next else None,
                                 _P(pm.data.data_ptr()), _P(xm.data_ptr()) if euler_coef is not None else None,
                                 _P(_ptr(out)), C.c_float(euler_coef or 0.0),
                                 _P(next_table.data_ptr()) if fused_next else None, C.byref(dims), stream)
        _native.check(rc, "lp_boundary")
        self.launches += 1
        return done

    # ---- CUDA-graph replay of a whole outer step -------------------------------------------------
    def _graphed_step(self, x, y, nz, pm, dims, table_np, tm_h, sigma_h, sigma_shape, active, plan, call_scaling,
                      model_options, seed):
        """Replay (capturing on first use) one CUDA graph holding the whole outer step: prologue,
        `active` x (model call + fused sub-step), final model call, epilogue.  Everything that changes
        between outer steps -- coefficient table, model timestep, sigma, RNG position -- lives in one
        small device block refreshed by a single H2D copy, so one graph serves every sigma of the
        schedule with the same sub-step count.  Returns None if capture is not possible (the caller
        then runs eagerly)."""
        dev = x.device
        B = x.shape[0]
        # what a captured graph bakes in besides the buffers: the launch geometry, everything the model read
        # from model_options, and the model object itself.  `seed` is handed to the model by value at capture;
        # none of ComfyUI's stock models consume it -- a model that does needs cuda_graph=False.
        key = (dev, tuple(x.shape), active, plan.mode, bool(call_scaling), tuple(sigma_shape),
               pm.row_stride, pm.channel_stride,
               id(self.inner_model) if self.graph_model_token is None else self.graph_model_token,
               options_fingerprint(model_options))
        g = self._graphs.get(key)
        if g is False:
            return None
        if g is None and self.graph_after > 0:
            # first sight of this configuration: run it eagerly (that IS the work; nothing is spent on a
            # warm-up pass) and capture when it comes back
            seen = self._graph_seen.get(key, 0)
            if seen < self.graph_after:
                self._graph_seen[key] = seen + 1
                return None
        st = self._graph_static(x, y, nz, pm, B)
        n_par = B * _native.TABLE_STRIDE + 2 * B + 4
        # ---- the dynamic block: [table | t_model | sigma | seed, base (2 x u64 in 4 float slots)] ----
        host = np.empty(n_par, dtype=np.float32)
        host[:B * _native.TABLE_STRIDE] = table_np.reshape(-1)
        o = B * _native.TABLE_STRIDE
        host[o:o + B] = tm_h
        host[o + B:o + 2 * B] = sigma_h
        host[o + 2 * B:].view(np.uint64)[:] = plan.state_words()
        if g is None:
            g = self._capture(key, st, dims, B, host, sigma_shape, active, plan, call_scaling, model_options, seed,
                              warm=self.graph_after <= 0)
            # keeps the ids inside the key from being recycled, and whatever the captured model call reads
            # through this guider (conditioning tensors) alive at the addresses the graph baked in
            self._graph_keep.append((model_options, self.inner_model))
            if g is None:
                self._graphs[key] = False
                return None
        g["params"].copy_(torch.from_numpy(host))
        st["x"].copy_(x)
        g["graph"].replay()
        self.launches += g["launches"]
        self.model_calls += g["model_calls"]
        plan.consume(g["draws"])
        x.copy_(st["x"])            # the in-place contract of lanpaint.py:156
        return g["out"].clone()     # a fresh tensor, like the reference returns

    def _graph_static(self, x, y, nz, pm, B):
        """Static operand buffers the graphs are captured against; refreshed when the source changes."""
        key = (x.device, tuple(x.shape))
        st = self._graph_statics.get(key)
        if st is None:
            st = {"x": torch.empty_like(x, dtype=torch.float32, memory_format=torch.contiguous_format),
                  "y": torch.empty_like(y), "nz": torch.empty_like(nz), "mask": torch.empty_like(pm.data),
                  "c": torch.empty_like(y), "src": [None, None, None]}
            while len(self._graph_statics) >= self.max_live_shapes:
                old = next(iter(self._graph_statics))
                self._graph_statics.pop(old)
                self._graphs = {k: g for k, g in self._graphs.items() if (k[0], k[1]) != old}
            self._graph_statics[key] = st
        for slot, (name, src) in enumerate((("y", y), ("nz", nz), ("mask", pm.data))):
            # inference tensors have no version counter: an in-place edit cannot be seen, so re-copy them
            if st["src"][slot] is None or not st["src"][slot].matches(src) or st["src"][slot].key[1] is None:
                if st[name].shape != src.shape:
                    st[name] = torch.empty_like(src)
                    self._graphs = {k: g for k, g in self._graphs.items() if (k[0], k[1]) != key}
                st[name].copy_(src)
                st["src"][slot] = _Ident(src)
        return st

    def _capture(self, key, st, dims, B, host, sigma_shape, active, plan, call_scaling, model_options, seed,
                 warm=True):
        dev = st["x"].device
        params = torch.from_numpy(host).to(dev)
        o = B * _native.TABLE_STRIDE
        tab = params[:o].view(B, _native.TABLE_STRIDE)
        t_model = params[o:o + B]
        sigma_dev = params[o + B:o + 2 * B].view(sigma_shape) if int(np.prod(sigma_shape)) == B else params[o + B:o + B + 1].view(sigma_shape)
        rng_state = params[o + 2 * B:].data_ptr()
        if rng_state % 8 != 0:
            return None
        out = torch.empty_like(st["x"])
        pm = PackedMask(st["mask"], key[6], key[7])
        rel = plan.relative()
        counts = (self.launches, self.model_calls)

        def body():
            rel.reset()
            self._launch_sequence(st["x"], st["y"], st["nz"], pm, dims, tab, t_model, sigma_dev, st["c"], out, active,
                                  rel, call_scaling, model_options, seed, None, rng_state)
        try:
            timer, self.kernel_timer = self.kernel_timer, None
            if warm:
                side = torch.cuda.Stream(device=dev)
                side.wait_stream(torch.cuda.current_stream(dev))
                with torch.cuda.stream(side):
                    body()  # warm-up outside capture: lazy inits, allocator
                torch.cuda.current_stream(dev).wait_stream(side)
            self.launches, self.model_calls = counts
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                body()
        except Exception as e:  # capture-unsafe model: run eagerly instead, say so once
            import warnings
            warnings.warn(f"lanpaint_b200: CUDA-graph capture failed ({type(e).__name__}: {e}); running eagerly")
            _repair_generator_after_failed_capture(dev)
            self.launches, self.model_calls = counts
            self.kernel_timer = timer
            return None
        self.kernel_timer = timer
        g = {"graph": graph, "params": params, "out": out, "draws": rel.used,
             "launches": self.launches - counts[0], "model_calls": self.model_calls - counts[1]}
        self.launches, self.model_calls = counts
        self._graphs[key] = g
        return g

    def _event_pair(self, flags):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        self.kernel_timer.append((flags, a, b))
        return a, b

    def _make_stopper(self, model_options, pm, like, abt_h, dims):
        semantic = model_options.get("lanpaint_semantic_stop") if isinstance(model_options, dict) else None
        if not (float(self.early_stop_threshold or 0.0) > 0.0 or isinstance(semantic, dict)):
            return None
        from .earlystop import make_stopper
        return make_stopper(model_options=model_options, default_threshold=self.early_stop_threshold,
                            default_patience=self.early_stop_patience, default_distance_fn=self.early_stop_hook,
                            packed_mask=pm, like=like, abt_mean=float(np.float32(abt_h.astype(np.float32).mean())),
                            dims=dims, reduce=self.stats_reduce)

    # ---- the reference's lower-level entry point, un-fused ------------------------------------------
    def langevin_dynamics(self, x_t, score, mask, step_size, current_times, sigma_x=1, sigma_y=0, args=None):
        """One Langevin sub-step around an arbitrary `score(x_t)` callback, in VP space, with the
        reference's signature and return value `(x_t, LangevinState(None, C, x0))`
        (src/LanPaint/lanpaint.py:192-293).  Because the callback sits between the two half-advances
        this cannot use the cross-model fusion: it runs lp_advance_f32 (first half), the callback, then
        lp_substep_f32 (Coef_C + correction + second half) -- 2 launches instead of ~89."""
        args = LangevinState.coerce(args)
        if not (isinstance(x_t, torch.Tensor) and x_t.is_cuda):
            raise RuntimeError("lanpaint_b200.LanPaint.langevin_dynamics needs CUDA tensors")
        lib = _native.load()
        dev = x_t.device
        B = x_t.shape[0]
        if self.img_dim_size is None:
            self.img_dim_size = x_t.ndim
        _, abt, _ = current_times

        def per_row(v):
            t = torch.as_tensor(v, dtype=torch.float32, device=dev).reshape(-1)
            return t if t.numel() == B else t[:1].expand(B)
        host = torch.stack([per_row(abt), per_row(step_size), per_row(sigma_x), per_row(sigma_y)]).cpu().numpy()
        abt_h, step_h, sx_h, sy_h = (host[k].astype(np.float64) for k in range(4))
        dt_free, dt_known = step_h * sx_h, step_h * sy_h       # the reference's dtx/2, dty/2 (lanpaint.py:301-328)
        if float(np.mean(dt_free.astype(np.float32))) <= 0.0:  # lanpaint.py:205
            return x_t, args
        table_np = np.empty((B, _native.TABLE_STRIDE), dtype=np.float32)
        rc = lib.lp_build_coef_table_dt(_P(abt_h.ctypes.data), None, _P(dt_free.ctypes.data), _P(dt_known.ctypes.data),
                                        C.c_double(float(self.chara_lamb)), 1, B, _P(table_np.ctypes.data))
        _native.check(rc, "lp_build_coef_table_dt")
        tab = torch.from_numpy(table_np).to(dev)
        pm = mask if isinstance(mask, PackedMask) else pack_mask(mask, x_t)
        per = x_t.numel() // B
        dims = _native.Dims(B, per, int(np.prod(x_t.shape[2:])) if x_t.ndim > 2 else 1, pm.row_stride, pm.channel_stride)
        stream = _P(_stream_ptr(dev))
        xt = _f32c(x_t).clone()
        first = args is None
        plan = _DrawPlan(self.rng, xt, 1 if first else 2)
        if first:
            cbuf = torch.empty_like(xt)
        else:
            cbuf = _f32c(args.C).clone()
            r = plan.rng_struct(1)
            rc = lib.lp_advance_f32(_P(xt.data_ptr()), _P(cbuf.data_ptr()), _P(pm.data.data_ptr()), _P(tab.data_ptr()),
                                    C.byref(dims), C.byref(r), 1, stream)
            _native.check(rc, "lp_advance_f32")
            self.launches += 1
        x0e_in = _f32c(xt + score(xt))                      # Coef_C's x0 = x_t + score(x_t), lanpaint.py:218
        x0e = torch.empty_like(xt)
        r = plan.rng_struct(1)
        flags = (_native.SUBSTEP_FIRST if first else 0) | _native.SUBSTEP_STORE_C
        rc = lib.lp_substep_f32(_P(xt.data_ptr()), _P(x0e_in.data_ptr()), _P(x0e_in.data_ptr()), _P(x0e_in.data_ptr()),
                                _P(pm.data.data_ptr()), _P(cbuf.data_ptr()), None, _P(x0e.data_ptr()),
                                _P(tab.data_ptr()), C.byref(dims), C.byref(r), flags, stream)
        _native.check(rc, "lp_substep_f32")
        self.launches += 1
        plan.finish()
        return xt.to(x_t.dtype), LangevinState(None, cbuf, x0e)

    # ---- MiniMax-H3 AV flat pack: trailing audio positions on their own schedule ----------------
    def _av_split(self, ai: torch.Tensor, n_last: int) -> int:
        """Validate that the indicator marks a suffix of the last axis and return where it starts
        (nodes.py:346: audio_indicator[..., video_n:] = 1).  One read-back per distinct indicator."""
        hit = self._av_cache.get(ai)
        if hit is not None:
            return hit
        flat = ai.reshape(-1, ai.shape[-1])
        if ai.shape[-1] != n_last or not bool((flat == flat[:1]).all()):
            raise NotImplementedError("audio_indicator must mark the same positions of the last axis on every row")
        line = (flat[0] > 0.5)
        split = int((~line).sum().item())
        if not bool(line[split:].all()) or bool(line[:split].any()):
            raise NotImplementedError("audio_indicator must be a suffix of the last axis (a flat AV pack)")
        self._av_cache.put(ai, split)
        return split

    def _av_blended_times(self, current_times, dev):
        """(VE, abt, flow_t) as the reference blends them for an AV pack (lanpaint.py:68-74); only built when
        an early-stop hook may read ctx["current_times"]."""
        VE, abt, flow_t = (t.to(dev) for t in current_times)
        VE_a, abt_a, _ = (t.to(dev) for t in self.current_times_audio)
        ai = self.audio_indicator.to(dev)
        return _blend(VE, VE_a, ai), _blend(abt, abt_a, ai), flow_t

    def _av_call(self, x, sigma, latent_mask, current_times, n_steps, model_options, seed, flow, opts):
        """lanpaint.py:60-74,173-180: audio positions take (VE, abt) and the replace sigma from the audio
        schedule and pull the model's target back by `audio_correction`; everything else is unchanged.
        Implemented with lp_dims.row_split: every row of the last axis has a second table row for its
        audio suffix, so the launches are the same single fused kernels."""
        rng = opts.get("rng", self.rng)
        dev = x.device
        if x.shape[0] != 1:
            raise NotImplementedError("AV per-row schedule needs batch 1 (the reference's broadcasting does too)")
        n_last = x.shape[-1]
        lines = x.numel() // n_last
        split = self._av_split(self.audio_indicator.to(dev), n_last)
        VE_Sigma, abt, Flow_t = current_times
        VE_a, abt_a, Flow_a = self.current_times_audio
        corr_t = self.audio_correction
        t_model_src = Flow_t if flow else VE_Sigma
        scal = [sigma, VE_Sigma, abt, t_model_src, VE_a, abt_a, Flow_a]
        vals = [t.reshape(-1)[:1].to(device=dev, dtype=torch.float32) for t in scal]
        if corr_t is not None:
            vals.append(corr_t.to(dev).reshape(-1)[-1:].float())   # an audio position (the last one)
        host = torch.cat(vals).cpu().numpy().astype(np.float64)
        s_v, ve_v, abt_v, tm_v, ve_au, abt_au, s_au = host[:7]
        c_au = float(host[7]) if corr_t is not None else 1.0
        hyper = Hyper(self.step_size, self.chara_lamb, self.chara_beta, self.min_step_frac, flow)
        ns = float(getattr(self.inner_model.inner_model.model_sampling, "noise_scale", 1.0))
        f32 = np.float32
        rep_n = [float(f32(s_v) * f32(ns))] * lines + [float(f32(s_au) * f32(ns))] * lines   # lanpaint.py:91-92
        rep_y = [float(f32(1.0) - f32(s_v))] * lines + [float(f32(1.0) - f32(s_au))] * lines
        table_np = build_table([abt_v] * lines + [abt_au] * lines, [ve_v] * lines + [ve_au] * lines, hyper,
                               rep_n, rep_y, [1.0] * lines + [c_au] * lines)
        if split == 0:   # an all-audio pack: row_split 0 means "no split", so every line reads the audio rows alone
            table_np = table_np[lines:]

        xm = x if (x.dtype == torch.float32 and x.is_contiguous()) else _f32c(x)
        y = _f32c(self.latent_image.to(dev))
        nz = _f32c(self.noise.to(dev))
        # the flat pack is indexed line by line (dims below): the mask becomes one uint8 per element
        if isinstance(latent_mask, PackedMask):      # what the node layer hands over (comfy_nodes._latent_mask)
            pm = self._av_mask_cache.get(latent_mask.data)
            if pm is None:
                data = latent_mask.data
                if data.numel() != x.numel():        # stored once per spatial site: repeat over the channels
                    data = data.expand(x.shape)
                pm = PackedMask(data.reshape(1, 1, -1).contiguous(), n_last, 0)
                self._av_mask_cache.put(latent_mask.data, pm)
        else:
            pm = self._mask_cache.get(latent_mask)
            if pm is None:
                full = latent_mask.to(dev).expand(x.shape)
                pm = pack_mask(full.reshape(1, 1, -1), xm.reshape(1, 1, -1))
                self._mask_cache.put(latent_mask, pm)
                self.launches += 1
        dims = _native.Dims(lines, n_last, n_last, n_last, 0, split)
        tab = torch.from_numpy(table_np).to(dev)
        t_model = t_model_src.reshape(-1).to(dev)
        present = ([abt_v] if split > 0 else []) + ([abt_au] if split < n_last else [])   # the schedules in use
        active = n_steps if mean_half_dt(present, hyper) > 0.0 else 0
        plan = _DrawPlan(rng, xm, active)
        out = torch.empty_like(xm)
        cbuf = torch.empty_like(xm)
        # lanpaint.py:104-111: the stopper sees the blended per-position abt; its mean is what scales the threshold
        abt_blend = np.float32((split * np.float32(abt_v) + (n_last - split) * np.float32(abt_au)) / n_last)
        flat = xm.reshape(1, 1, -1)
        stopper = self._make_stopper(model_options, pm, flat, np.asarray([abt_blend]), dims)
        times_blend = (VE_Sigma, abt, Flow_t) if stopper is None else self._av_blended_times(current_times, dev)
        done = self._launch_sequence(xm, y, nz, pm, dims, tab, t_model, sigma.to(dev), cbuf, out, active, plan, False,
                                     model_options, seed, stopper, None, current_times=times_blend)
        plan.finish()
        self.substeps_done += done
        if xm is not x:
            x.copy_(xm)
        return out if out.dtype == x.dtype else out.to(x.dtype)


def _blend(a, b, ai):
    return a * (1 - ai) + b * ai


def _repair_generator_after_failed_capture(dev: torch.device) -> None:
    """A capture that dies between capture_begin and capture_end leaves torch's default CUDA generator
    flagged as "capturing" (every later torch.rand* then raises "Offset increment outside graph
    capture").  Swapping in a cloned state object clears the flag and keeps seed and offset."""
    try:
        torch.cuda.synchronize(dev)
    except Exception:
        pass
    try:
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        gen = torch.cuda.default_generators[idx]
        gen.graphsafe_set_state(gen.clone_state())
    except Exception:
        pass


_HEAD_DTYPES = {torch.float32: _native.DTYPE_F32, torch.bfloat16: _native.DTYPE_BF16, torch.float16: _native.DTYPE_F16}


def _as_operand(t: torch.Tensor, like: torch.Tensor) -> torch.Tensor:
    """A model output as a kernel operand: latent shape, contiguous, fp32 / bf16 / fp16 kept as is (the kernels
    widen half-precision heads in registers, the values type promotion gives the reference at lanpaint.py:182-184);
    anything else is converted to fp32."""
    if not isinstance(t, torch.Tensor):
        raise TypeError(f"model returned {type(t).__name__}, expected a tensor")
    if t.shape != like.shape:
        t = t.expand(like.shape)
    if t.device != like.device:
        t = t.to(like.device)
    if t.dtype not in _HEAD_DTYPES:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


def _heads(a: torch.Tensor, b: Optional[torch.Tensor], like: torch.Tensor, combine: bool = False, cfg: float = 0.0,
           cfg_big: float = 0.0, dead: bool = False):
    """-> (lp_heads struct, tensors to keep alive).  a / b end up with one common dtype.  dead: LP_HEADS_DEAD."""
    a = _as_operand(a, like)
    b = a if (b is None or b is a) else _as_operand(b, like)
    if b.dtype != a.dtype or (combine and a.dtype != torch.float32):
        a, b = a.float(), (a.float() if b is a else b.float())
    h = _native.Heads(a.data_ptr(), b.data_ptr(), _HEAD_DTYPES[a.dtype] | (_native.HEADS_DEAD if dead else 0),
                      1 if combine else 0, float(cfg), float(cfg_big))
    return h, (a, b)


def heads_discardable(model_options) -> bool:
    """Whether a job that owns its network calls may let the update kernels discard the network's outputs once read
    (`_launch_sequence(discard_heads=True)`): not when a user CFG hook has seen them (ComfyUI's sampler_cfg_function
    / sampler_post_cfg_function receive the raw predictions and may keep them), nor when the network re-reads its
    own output and says so with the option {"discard_heads": False}."""
    mo = model_options or {}
    if not (mo.get("lanpaint_b200") or {}).get("discard_heads", True):
        return False
    return "sampler_cfg_function" not in mo and not mo.get("sampler_post_cfg_function")


def _probe_noise_scaling(sampling, sigma: float):
    """Recover (a, b) with noise_scaling(sigma, n, y) == a*n + b*y from four host
    probe points; None if the function is not of that form (or misbehaves)."""
    try:
        s = torch.tensor([[sigma]], dtype=torch.float32)
        n = torch.tensor([[1.0, 0.0, 1.0, 2.0]], dtype=torch.float32)
        y = torch.tensor([[0.0, 1.0, 1.0, -3.0]], dtype=torch.float32)
        r = sampling.noise_scaling(s, n.clone(), y.clone())
        r = r.reshape(-1).double().tolist()
    except Exception:
        return None
    if len(r) != 4:
        return None
    a, b = r[0], r[1]
    tol = 1e-5 * (abs(a) + abs(b) + 1.0)
    if abs(r[2] - (a + b)) > tol or abs(r[3] - (2 * a - 3 * b)) > tol:
        return None
    return a, b


class _DrawPlan:
    """Maps the reference's sequence of randn_like draws onto kernel launches."""

    def __init__(self, rng, like: torch.Tensor, n_steps: int):
        self.rng = rng
        self.like = like
        self.n_draws = 0 if n_steps <= 0 else 2 * n_steps - 1
        self.used = 0
        self.gen = None
        self.inc = 4
        if isinstance(rng, NoiseTape):
            self.mode = _native.RNG_TAPE
        elif rng in ("torch", "philox"):
            self.mode = _native.RNG_TORCH if rng == "torch" else _native.RNG_PHILOX
            idx = like.device.index if like.device.index is not None else torch.cuda.current_device()
            self.gen = torch.cuda.default_generators[idx]
            self.seed = int(self.gen.initial_seed()) & 0xFFFFFFFFFFFFFFFF
            self.offset = int(self.gen.get_offset())
            if self.mode == _native.RNG_TORCH:
                g, inc = C.c_int64(0), C.c_uint64(0)
                rc = _native.load().lp_torch_randn_geometry(like.numel(), idx, C.byref(g), C.byref(inc))
                _native.check(rc, "lp_torch_randn_geometry")
                self.inc = int(inc.value)
        else:
            raise ValueError(f"unknown rng {rng!r}: use 'torch', 'philox' or a NoiseTape")
        self._keep: List[torch.Tensor] = []

    def rng_struct(self, k: int, state_ptr=None) -> _native.Rng:
        """rng argument of a launch that consumes the next k (1 or 2) draws.  With `state_ptr`
        (graph capture) the positions are relative to the {seed, base} block the kernel reads."""
        r = _native.Rng()
        r.mode = self.mode
        if self.mode == _native.RNG_TAPE:
            t0 = self.rng.next(self.like)
            t1 = self.rng.next(self.like) if k == 2 else None
            self._keep = [t0, t1]
            r.tape0 = t0.data_ptr()
            r.tape1 = None if t1 is None else t1.data_ptr()
        else:
            rel = state_ptr is not None
            r.seed = 0 if rel else self.seed
            r.state = state_ptr
            step = self.inc if self.mode == _native.RNG_TORCH else 1
            base = 0 if rel else (self.offset if self.mode == _native.RNG_TORCH else self.offset // 4)
            r.draw0 = base + self.used * step
            r.draw1 = base + (self.used + 1) * step
        self.used += k
        return r

    def relative(self):
        """A plan used while capturing: counts draws from zero, touches no generator."""
        p = object.__new__(_DrawPlan)
        p.__dict__.update(self.__dict__)
        p.gen = None
        p.used = 0
        return p

    def reset(self):
        self.used = 0

    def consume(self, k: int):
        self.used += k

    def state_words(self):
        """{seed, base} as the kernels read them through lp_rng.state."""
        base = self.offset if self.mode == _native.RNG_TORCH else self.offset // 4
        return np.array([self.seed, base], dtype=np.uint64)

    def finish(self):
        """Advance the global generator by what the reference would have consumed."""
        if self.gen is not None and self.used:
            self.gen.set_offset(self.offset + self.used * self.inc)
