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
