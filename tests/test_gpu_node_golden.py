"""GPU: the four sampler nodes, LATENT dict in -> LATENT dict out, against outputs of the REFERENCE's own node layer.

The fixtures (`tests/golden/node_*.npz`, written by `tests/golden/make_node_golden.py`) come from the unmodified
reference `src/LanPaint/nodes.py` driven on the CPU over minicomfy with `torch.randn_like` on a recorded tape.
Here the same call goes through `lanpaint_b200.comfy_nodes` on the GPU with that tape as the engine's Gaussian
stream (and as `torch.randn_like` for the draws the node layer / an ancestral sampler make themselves), so what is
compared is everything between the two LATENT dicts: mask preparation, noise scaling, the sigma -> (VE, abt, t)
glue, the inner-step ramp, dual CFG, the fused update kernels, the sampler's own steps and the epilogue
(nodes.py:161-216, 229-379, 487-513).  Tolerance: the north_star contract (1e-3 of the final latent's scale)
with fp32 round-off asserted at 5e-6 (the network stand-in's tanh differs by an ulp between CPU and GPU).  `node_av_flat_pack` enters at the patched CFGGuider.outer_sample with `latent_shapes`, the way ComfyUI
hands over a nested (video, audio) latent (MiniMax-H3: audio rows on their own shifted sigma schedule).
The `*_mix` fixtures run the same calls with `_node_cases.mixing_denoiser`, a network that couples positions, so that
what the node layer does at known positions (cfg_BIG, lambda, the replace step, the noise image) reaches `out`."""
import glob
import json
import os
import sys
from unittest import mock

import numpy as np
import pytest
import torch

import minicomfy
from _node_cases import build_patcher, call_node, net_of
from _support import max_rel
from conftest import GOLDEN_DIR

pytestmark = pytest.mark.gpu

NODE_CASES = sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(GOLDEN_DIR, "node_*.npz")))
CONTRACT = 1e-3        # BASELINE.json north_star: relative fp32 on the final latent
EXPECTED = 5e-6        # fp32 round-off through a whole sampler run
_MEASURED = {}


def load_node_golden(name):
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    g = {k: z[k] for k in z.files if k != "meta"}
    g["meta"] = json.loads(str(z["meta"]))
    return g


def test_fixture_inventory():
    assert len(NODE_CASES) >= 13
    nodes = {load_node_golden(n)["meta"]["node"] for n in NODE_CASES}
    assert nodes == {"LanPaint_KSampler", "LanPaint_KSamplerAdvanced", "LanPaint_SamplerCustom",
                     "LanPaint_SamplerCustomAdvanced", "outer_sample_av_pack"}


@pytest.mark.parametrize("name", NODE_CASES)
def test_node_matches_reference_node_layer(name, cuda_device):
    minicomfy.install()
    from lanpaint_b200 import comfy_nodes as N
    from lanpaint_b200.engine import NoiseTape
    g = load_node_golden(name)
    c = g["meta"]
    dev = cuda_device
    calls = {"n": 0}

    def net(x, sigma, cond):
        calls["n"] += 1
        return net_of(c)(x, sigma, cond)

    patcher = build_patcher(c, device=dev, net=net)
    tape = NoiseTape([torch.from_numpy(t.astype(np.float32)) for t in g["tape"]])
    # the tape is the engine's Gaussian stream; plain launches (a tape cannot be replayed from a captured graph)
    # (and ComfyUI's CPU noise image comes from the fixture, not from the device-side draw of this host's stream)
    patcher.model_options["lanpaint_b200"] = {"rng": tape, "cuda_graph": False, "device_noise": False}
    latent = {"samples": torch.from_numpy(g["samples"])}
    if "noise_mask" in g:
        latent["noise_mask"] = torch.from_numpy(g["noise_mask"].astype(np.float32))
    noise_image = torch.from_numpy(g["noise_image"]) if "noise_image" in g else None

    def prepare_noise(latent_image, seed, noise_inds=None):     # ComfyUI's CPU randn, as the reference run saw it
        return noise_image.clone()

    def randn_like(like, **kwargs):                              # Noise_RandomNoise / an ancestral sampler
        return tape.next(like)

    comfy_sample = sys.modules["comfy.sample"]
    with mock.patch.object(comfy_sample, "prepare_noise", prepare_noise), mock.patch.object(torch, "randn_like", randn_like):
        outs = call_node(N, c, patcher, latent, noise_image)

    assert tape.pos == c["n_draws"], "draw count / order differs from the reference's node layer"
    assert calls["n"] == c["network_calls"], "number of network evaluations differs from the reference's"
    assert float(patcher.LanPaint_cfg_BIG) == c["cfg_big"]
    out = outs[0]["samples"]
    assert out.device.type == "cpu" and tuple(out.shape) == tuple(g["out"].shape)
    err = max_rel(out, torch.from_numpy(g["out"]))
    _MEASURED[name] = err
    if "denoised_out" in g:
        assert len(outs) == 2
        err_d = max_rel(outs[1]["samples"], torch.from_numpy(g["denoised_out"]))
        _MEASURED[name + ":denoised"] = err_d
        assert err_d <= CONTRACT, err_d
    if "noise_mask" in latent:
        assert "noise_mask" in outs[0]
    assert err <= CONTRACT, err
    assert err <= EXPECTED, f"{name}: {err:.3e} is inside the 1e-3 contract but above fp32 round-off"


@pytest.mark.parametrize("name", NODE_CASES)
def test_engine_seam_under_the_reference_node_layer(name, cuda_device, monkeypatch):
    """INTEGRATION.md seam 2, literally: the REFERENCE's own node layer (oracle/_ref bytecode of nodes.py: its patch
    seam, its per-sigma wrapper with device-resident sigma / current_times and a full-shape fp32 latent_mask) with the
    one-line engine swap `LanPaint = lanpaint_b200.engine.LanPaint` (nodes.py:18), on the GPU, against the outputs the
    same node layer produced with the reference's engine."""
    import contextlib
    import io
    from oracle import build_ref
    ref_nodes = build_ref.load_nodes()
    if ref_nodes is None:
        pytest.skip("oracle/_ref not built (needs /root/reference: `make -C oracle`)")
    from lanpaint_b200.engine import LanPaint, NoiseTape
    monkeypatch.setattr(ref_nodes, "LanPaint", LanPaint)
    g = load_node_golden(name)
    c = g["meta"]
    dev = cuda_device
    calls = {"n": 0}

    def net(x, sigma, cond):
        calls["n"] += 1
        return net_of(c)(x, sigma, cond)

    patcher = build_patcher(c, device=dev, net=net)
    tape = NoiseTape([torch.from_numpy(t.astype(np.float32)) for t in g["tape"]])
    patcher.model_options["lanpaint_b200"] = {"rng": tape}
    latent = {"samples": torch.from_numpy(g["samples"])}
    if "noise_mask" in g:
        latent["noise_mask"] = torch.from_numpy(g["noise_mask"].astype(np.float32))
    noise_image = torch.from_numpy(g["noise_image"]) if "noise_image" in g else None
    comfy_sample = sys.modules["comfy.sample"]
    with mock.patch.object(comfy_sample, "prepare_noise", lambda *a, **k: noise_image.clone()), \
            mock.patch.object(torch, "randn_like", lambda like, **kw: tape.next(like)), \
            contextlib.redirect_stdout(io.StringIO()):
        outs = call_node(ref_nodes, c, patcher, latent, noise_image)
    assert tape.pos == c["n_draws"] and calls["n"] == c["network_calls"]
    err = max_rel(outs[0]["samples"], torch.from_numpy(g["out"]))
    _MEASURED[name + ":reference-nodes+b200-engine"] = err
    assert err <= EXPECTED, err


def test_report_measured_errors():
    """Prints the measured deviations."""
    if not _MEASURED:
        pytest.skip("no node case ran")
    print("node-level max |out - reference| / max|reference|:", json.dumps(_MEASURED, sort_keys=True))
    assert max(_MEASURED.values()) <= CONTRACT
