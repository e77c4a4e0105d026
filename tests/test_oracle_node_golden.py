"""CPU: the oracle's restatement of the node-level glue (`euler_inpaint`: noise scaling, sigma -> times, inner-step
ramp, dual CFG, Euler steps -- nodes.py:161-175, 229-315, 319-379) against outputs of the REFERENCE's own node
layer (`tests/golden/node_*.npz`, see tests/golden/make_node_golden.py).  This is what pins the oracle above the
engine seam: the GPU node tests that compare with `O.euler_inpaint` inherit it."""
import json
import os

import numpy as np
import pytest
import torch

import minicomfy
from _node_cases import NEG, POS, net_of
from conftest import GOLDEN_DIR
from oracle import langevin_oracle as O

EULER_KSAMPLER_CASES = ["node_ksampler_sdxl_karras20_n5", "node_ksampler_prompt_first_batch2", "node_ksampler_flux_simple"]
# the same calls with a network that couples positions: pins the oracle's glue at known positions as well
EULER_KSAMPLER_CASES += [n + "_mix" for n in EULER_KSAMPLER_CASES]


class _Guider:
    """What the reference's patched CFGGuider hands the engine: (x0 at cfg, x0 at cfg_BIG), nodes.py:161-175;
    at cfg == 1 ComfyUI skips the uncond evaluation and the combine returns cond itself."""

    def __init__(self, sampling, cfg, cfg_big, net):
        self.inner_model, self.model_sampling, self.cfg, self.cfg_big, self.calls = self, sampling, cfg, cfg_big, 0
        self.net = net

    def __call__(self, x, sigma, model_options=None, seed=None):
        c = self.net(x, sigma, POS)
        self.calls += 1
        if self.cfg == 1.0:
            u = c
        else:
            u = self.net(x, sigma, NEG)
            self.calls += 1
        return u + (c - u) * self.cfg, u + (c - u) * self.cfg_big


@pytest.mark.parametrize("name", EULER_KSAMPLER_CASES)
def test_oracle_euler_run_equals_reference_node_run(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    c = json.loads(str(z["meta"]))
    a = c["args"]
    flow = c.get("model_type", "EPS") in ("FLUX", "FLOW")
    y = torch.from_numpy(z["samples"])
    noise = torch.from_numpy(z["noise_image"])
    dm = torch.from_numpy(z["noise_mask"].astype(np.float32))
    dm = minicomfy.repeat_to_batch_size(dm, y.shape[0]).expand(y.shape)       # same-resolution masks only here
    base = minicomfy.BaseModel(net_of(c), model_type=getattr(minicomfy.ModelType, c.get("model_type", "EPS")),
                               latent_channels=y.shape[1], shift=c.get("shift", 1.0))
    sig = minicomfy.KSampler(minicomfy.ModelPatcher(base, "cpu"), a["steps"], "cpu", a["sampler_name"],
                             a["scheduler"]).sigmas
    model = _Guider(O.FlowSampling() if flow else O.VESampling(), a["cfg"], c["cfg_big"], net_of(c))
    tape = O.NoiseTape([torch.from_numpy(t.astype(np.float32)) for t in z["tape"]])
    cnt = {}
    with torch.no_grad():
        got = O.euler_inpaint(model, y, noise, dm, sig, O.Hyper(n_steps=a["LanPaint_NumSteps"], min_step_frac=1.0, flow=flow),
                              draw=tape, max_denoise=not flow, counters=cnt)
        got = base.model_sampling.inverse_noise_scaling(sig[-1], got)
    assert tape.pos == c["n_draws"] and model.calls == c["network_calls"]
    want = torch.from_numpy(z["out"])
    err = float((got - want).abs().max() / want.abs().max())
    assert err <= 1e-6, err


# ---------------------------------------------------------------------------------------------------------------
# `_job_ref.job` (the loop the GPU job tests run in fp64) on the routes outside the plain Euler KSampler
# ---------------------------------------------------------------------------------------------------------------
JOB_CASES = ["node_ksampler_heun_mix", "node_ksampler_ancestral", "node_advanced_window_leftover_mix",
             "node_advanced_noise_disabled_mix", "node_custom_random_noise_mix", "node_custom_advanced",
             "node_av_flat_pack_mix"]


def fixture_job(z, dtype=torch.float32):
    """Runs `_job_ref.job` on a node fixture's inputs and tape: (out, the last step's denoised latent, tape, model).
    Every node argument becomes a job input: the schedule, max_denoise, lambda, step size and cfg_BIG, the noise
    image (zero for add_noise = disable; the tape's first draw for SamplerCustom's Noise_RandomNoise), the audio
    rows of an AV pack."""
    import _job_ref as J
    c = json.loads(str(z["meta"]))
    a = c["args"]
    mtype = c.get("model_type", "EPS")
    flow = mtype in ("FLUX", "FLOW")
    y = torch.from_numpy(z["samples"]).to(dtype)
    dm = torch.from_numpy(z["noise_mask"].astype(np.float32))
    if dm.shape != y.shape:                 # a latent-resolution mask, broadcast over channels and batch
        dm = minicomfy.repeat_to_batch_size(dm, y.shape[0]).expand(y.shape)
    base = minicomfy.BaseModel(net_of(c), model_type=getattr(minicomfy.ModelType, mtype), latent_channels=y.shape[1],
                               shift=c.get("shift", 1.0))
    tape = O.NoiseTape([torch.from_numpy(t.astype(np.float32)) for t in z["tape"]])
    audio, node = None, c["node"]
    if node in ("LanPaint_KSampler", "LanPaint_KSamplerAdvanced"):
        sampler = a["sampler_name"]
        window = {}
        if node == "LanPaint_KSamplerAdvanced":
            window = dict(start_step=a["start_at_step"], last_step=a["end_at_step"],
                          force_full_denoise=a["return_with_leftover_noise"] != "enable")
        sig = J.ksampler_sigmas(minicomfy.ModelPatcher(base, "cpu"), a["steps"], sampler, a["scheduler"],
                                a.get("denoise", 1.0), **window)
        noise = torch.zeros_like(y) if a.get("add_noise") == "disable" else torch.from_numpy(z["noise_image"])
    elif node == "outer_sample_av_pack":
        sampler, sig = "euler", torch.tensor(a["sigmas"], dtype=torch.float32)
        noise = torch.from_numpy(z["noise_image"])
        audio = J.av_audio(a["n_video"], a["shift_video"], a["shift_audio"])
    else:
        sampler, (_, n) = a["sampler"], a["sigmas"]
        sig = minicomfy.get_sigmas_karras(n, 0.0292, 14.6146)
        if node == "LanPaint_SamplerCustom":
            noise = tape(y) if a["add_noise"] else torch.zeros_like(y)
        else:
            noise = torch.from_numpy(z["noise_image"])
    hp = O.Hyper(n_steps=a["LanPaint_NumSteps"], lam=a.get("LanPaint_Lambda", 5.0),
                 step_size=a.get("LanPaint_StepSize", 0.2), min_step_frac=1.0, flow=flow)
    model = J.Guider(net_of(c), O.FlowSampling() if flow else O.VESampling(), a["cfg"],
                     1.0 if mtype == "FLUX" else c["cfg_big"])
    steps = []
    got = J.job(J.SAMPLERS[sampler], model, y, noise.to(dtype), dm.to(dtype), sig, hp, draw=tape,
                max_denoise=J.max_denoise(base.model_sampling, sig[0]), callback=lambda i, d: steps.append(d),
                audio=audio)
    return got, steps[-1], tape, model


@pytest.mark.parametrize("name", JOB_CASES)
def test_job_loop_reproduces_reference_node_run(name):
    """The fp32 job on a fixture's tape == the reference node layer's outputs, draw for draw and call for call."""
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    c = json.loads(str(z["meta"]))
    got, denoised, tape, model = fixture_job(z)
    assert tape.pos == c["n_draws"], (tape.pos, c["n_draws"])
    assert model.calls == c["network_calls"], (model.calls, c["network_calls"])
    for key, g in (("out", got), ("denoised_out", denoised)):
        if key in z.files:
            want = torch.from_numpy(z[key])
            err = float((g - want).abs().max() / want.abs().max())
            assert err <= 1e-6, (key, err)
