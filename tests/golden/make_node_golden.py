"""Node-level golden vectors from the REAL reference node layer (run in the build container only).

    python tests/golden/make_node_golden.py                  # writes tests/golden/node_*.npz
    python tests/golden/make_node_golden.py --only '_mix$'   # writes only the fixtures whose name matches

The unmodified `/root/reference/src/LanPaint/nodes.py` is imported with `minicomfy` standing in for ComfyUI and
its four sampler nodes are driven on the CPU, from the LATENT dict in to the LATENT dict out: common_ksampler /
sample_custom -> the reference's patched CFGGuider.outer_sample / predict_noise -> its KSAMPLER.sample -> its
per-sigma wrapper (nodes.py:229-315) -> `LanPaint.__call__`.  `torch.randn_like` -- every Gaussian draw of the
Langevin loop (lanpaint.py:252), of `Noise_RandomNoise` (nodes.py:666-671) and of an ancestral sampler -- is patched
to a recording tape whose values are exactly representable in fp16 (so the tape is stored as fp16, bit for bit).

Each fixture carries what a node-level parity test needs: the LATENT dict (`samples`, `noise_mask`), the JSON
arguments of the call, the noise image ComfyUI's CPU `prepare_noise` produced (its bits depend on the host's CPU
dispatch, so tests feed it back instead of re-drawing it), the tape, the number of network evaluations, and the
node's outputs.  `/root/reference` does not exist on the GPU box: nothing but this script reads it.
"""
from __future__ import annotations

import importlib
import json
import os
import re
import sys
import warnings
from unittest import mock

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, "/root/reference")

sys.path.insert(0, os.path.join(ROOT, "tests"))

import minicomfy  # noqa: E402
from _node_cases import (FixedNoise, IMAGE_MODE, NEG, POS, VIDEO_MODE, build_patcher, call_node,  # noqa: E402
                         net_of)


class Fp16Tape:
    """Stand-in for torch.randn_like: N(0,1) draws rounded to fp16-representable values, recorded in order."""

    def __init__(self, seed):
        self.g = torch.Generator().manual_seed(seed)
        self.recorded = []

    def __call__(self, like, **kwargs):
        t = torch.randn(like.shape, generator=self.g, dtype=torch.float32).half().float()
        self.recorded.append(t)
        return t.to(device=like.device, dtype=like.dtype)


# name, node, latent shape, mask shape, model type / class, the node's own arguments
CASES = [
    dict(name="node_ksampler_sdxl_karras20_n5", node="LanPaint_KSampler", shape=(1, 4, 16, 16), mask=(1, 1, 16, 16),
         args=dict(seed=3, steps=20, cfg=5.0, sampler_name="euler", scheduler="karras", denoise=1.0,
                   LanPaint_NumSteps=5, LanPaint_PromptMode="Image First", Inpainting_mode=IMAGE_MODE)),
    dict(name="node_ksampler_prompt_first_batch2", node="LanPaint_KSampler", shape=(2, 4, 8, 8), mask=(1, 1, 8, 8),
         args=dict(seed=11, steps=8, cfg=6.5, sampler_name="euler", scheduler="karras", denoise=1.0,
                   LanPaint_NumSteps=3, LanPaint_PromptMode="Prompt First", Inpainting_mode=IMAGE_MODE)),
    dict(name="node_ksampler_pixel_mask", node="LanPaint_KSampler", shape=(1, 4, 8, 8), mask=(1, 64, 64),
         args=dict(seed=5, steps=6, cfg=4.0, sampler_name="euler", scheduler="karras", denoise=1.0,
                   LanPaint_NumSteps=2, LanPaint_PromptMode="Image First", Inpainting_mode=IMAGE_MODE)),
    dict(name="node_ksampler_flux_simple", node="LanPaint_KSampler", shape=(1, 16, 8, 8), mask=(1, 1, 8, 8),
         model_type="FLUX", shift=1.15,
         args=dict(seed=21, steps=10, cfg=1.0, sampler_name="euler", scheduler="simple", denoise=1.0,
                   LanPaint_NumSteps=3, LanPaint_PromptMode="Image First", Inpainting_mode=IMAGE_MODE)),
    dict(name="node_ksampler_flow_video", node="LanPaint_KSampler", shape=(1, 16, 3, 4, 4), mask=(9, 1, 32, 32),
         model_type="FLOW", shift=3.0, wan22=True,
         args=dict(seed=8, steps=8, cfg=3.5, sampler_name="euler", scheduler="simple", denoise=1.0,
                   LanPaint_NumSteps=3, LanPaint_PromptMode="Image First", Inpainting_mode=VIDEO_MODE)),
    dict(name="node_ksampler_heun", node="LanPaint_KSampler", shape=(1, 4, 8, 8), mask=(1, 1, 8, 8),
         args=dict(seed=2, steps=6, cfg=5.0, sampler_name="heun", scheduler="karras", denoise=1.0,
                   LanPaint_NumSteps=2, LanPaint_PromptMode="Image First", Inpainting_mode=IMAGE_MODE)),
    dict(name="node_ksampler_ancestral", node="LanPaint_KSampler", shape=(1, 4, 8, 8), mask=(1, 1, 8, 8),
         args=dict(seed=9, steps=6, cfg=5.0, sampler_name="euler_ancestral", scheduler="karras", denoise=1.0,
                   LanPaint_NumSteps=2, LanPaint_PromptMode="Image First", Inpainting_mode=IMAGE_MODE)),
    dict(name="node_ksampler_no_mask", node="LanPaint_KSampler", shape=(1, 4, 8, 8), mask=None,
         args=dict(seed=4, steps=5, cfg=5.0, sampler_name="euler", scheduler="karras", denoise=1.0,
                   LanPaint_NumSteps=2, LanPaint_PromptMode="Image First", Inpainting_mode=IMAGE_MODE)),
    dict(name="node_advanced_window_leftover", node="LanPaint_KSamplerAdvanced", shape=(1, 4, 8, 8), mask=(1, 1, 8, 8),
         args=dict(add_noise="enable", noise_seed=13, steps=12, cfg=5.0, sampler_name="euler", scheduler="karras",
                   start_at_step=2, end_at_step=9, return_with_leftover_noise="enable", LanPaint_NumSteps=2,
                   LanPaint_Lambda=8.0, LanPaint_StepSize=0.15, LanPaint_PromptMode="Image First",
                   Inpainting_mode=IMAGE_MODE)),
    dict(name="node_advanced_noise_disabled", node="LanPaint_KSamplerAdvanced", shape=(1, 4, 8, 8), mask=(1, 1, 8, 8),
         args=dict(add_noise="disable", noise_seed=1, steps=6, cfg=5.0, sampler_name="euler", scheduler="karras",
                   start_at_step=2, end_at_step=10000, return_with_leftover_noise="disable", LanPaint_NumSteps=2,
                   LanPaint_Lambda=5.0, LanPaint_StepSize=0.2, LanPaint_PromptMode="Prompt First",
                   Inpainting_mode=IMAGE_MODE)),
    dict(name="node_custom_random_noise", node="LanPaint_SamplerCustom", shape=(2, 4, 8, 8), mask=(2, 1, 8, 8),
         args=dict(add_noise=True, noise_seed=17, cfg=7.0, sampler="euler", sigmas=("karras", 7),
                   LanPaint_NumSteps=3, LanPaint_PromptMode="Image First")),
    dict(name="node_custom_advanced", node="LanPaint_SamplerCustomAdvanced", shape=(1, 4, 8, 8), mask=(1, 1, 8, 8),
         args=dict(noise_seed=23, cfg=4.0, sampler="euler", sigmas=("karras", 8), LanPaint_NumSteps=3,
                   LanPaint_Lambda=6.0, LanPaint_StepSize=0.25, LanPaint_PromptMode="Prompt First")),
    # MiniMax-H3 AV flat pack [1, C, video_n + audio_n]: the audio rows run on their own shifted sigma schedule
    dict(name="node_av_flat_pack", node="outer_sample_av_pack", shape=(1, 8, 128), mask=(1, 8, 128), model_type="FLOW",
         args=dict(seed=2, cfg=1.0, sigmas=[0.95, 0.8, 0.6, 0.4, 0.2, 0.0], LanPaint_NumSteps=3, n_video=96, n_audio=32,
                   shift_video=3.0, shift_audio=1.5)),
]


# the same calls with a network that couples positions (`_node_cases.mixing_denoiser`): only with it do the settings
# that act at known positions (cfg_BIG / prompt mode, lambda, the noise image, add_noise) reach the output latent
MIXED = ("node_ksampler_sdxl_karras20_n5", "node_ksampler_prompt_first_batch2", "node_ksampler_flux_simple",
         "node_ksampler_flow_video", "node_ksampler_heun", "node_advanced_window_leftover", "node_advanced_noise_disabled",
         "node_custom_random_noise", "node_av_flat_pack")
CASES += [dict(c, name=c["name"] + "_mix", net="mixing") for c in CASES if c["name"] in MIXED]


def case_inputs(c):
    g = torch.Generator().manual_seed(100 + len(c["name"]))
    y = torch.randn(c["shape"], generator=g)
    latent = {"samples": y}
    if c["mask"] is not None:
        latent["noise_mask"] = (torch.rand(c["mask"], generator=g) < 0.5).float()     # 1 = regenerate
    return latent


def main(argv=None):
    import argparse
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--only", metavar="REGEX", help="write only the fixtures whose name matches (re.search); the "
                    "others stay untouched (rewriting one changes its zip timestamps even when the arrays do not)")
    args = ap.parse_args(argv)
    warnings.filterwarnings("ignore")
    torch.set_num_threads(1)
    minicomfy.install()
    ref = importlib.import_module("src.LanPaint.nodes")
    assert ref.__file__.startswith("/root/reference/"), ref.__file__
    real_prepare_noise = minicomfy.prepare_noise
    for c in CASES:
        if args.only is not None and not re.search(args.only, c["name"]):
            continue
        latent = case_inputs(c)
        calls = {"n": 0}

        def net(x, sigma, cond):
            calls["n"] += 1
            return net_of(c)(x, sigma, cond)

        patcher = build_patcher(c, net=net)
        tape = Fp16Tape(seed=4321 + len(c["name"]))
        noise_images = []

        def prepare_noise(latent_image, seed, noise_inds=None):
            noise_images.append(real_prepare_noise(latent_image, seed, noise_inds))
            return noise_images[-1]

        fixed = None
        if c["node"] in ("LanPaint_SamplerCustomAdvanced", "outer_sample_av_pack"):
            fixed = torch.randn(c["shape"], generator=torch.Generator().manual_seed(c["args"].get("noise_seed", 77)))
            noise_images.append(fixed)
        sys.modules["comfy.sample"].prepare_noise = prepare_noise
        try:
            with mock.patch.object(torch, "randn_like", tape), open(os.devnull, "w") as devnull:
                stdout, sys.stdout = sys.stdout, devnull        # the reference prints from outer_sample
                try:
                    outs = call_node(ref, c, patcher, dict(latent), fixed)
                finally:
                    sys.stdout = stdout
        finally:
            sys.modules["comfy.sample"].prepare_noise = real_prepare_noise
        shape = tuple(c["shape"])
        assert all(tuple(t.shape) == shape for t in tape.recorded), "a draw of another shape: extend the fixture format"
        arrays = dict(samples=latent["samples"].numpy(),
                      tape=(np.stack([t.numpy() for t in tape.recorded]).astype(np.float16) if tape.recorded
                            else np.zeros((0,) + shape, np.float16)),
                      out=outs[0]["samples"].numpy())
        if "noise_mask" in latent:
            arrays["noise_mask"] = latent["noise_mask"].numpy().astype(np.uint8)
        if noise_images:
            arrays["noise_image"] = noise_images[0].numpy()
        if len(outs) > 1:
            arrays["denoised_out"] = outs[1]["samples"].numpy()
        meta = dict(c, n_draws=len(tape.recorded), network_calls=calls["n"], pos=POS, neg=NEG,
                    cfg_big=float(patcher.LanPaint_cfg_BIG),
                    generator="reference@/root/reference src/LanPaint/nodes.py over minicomfy, CPU, 1 thread")
        np.savez_compressed(os.path.join(HERE, c["name"] + ".npz"), meta=np.array(json.dumps(meta, ensure_ascii=False)),
                            **arrays)
        print(f"{c['name']:38s} draws={len(tape.recorded):3d} network calls={calls['n']:3d} "
              f"|out|={float(outs[0]['samples'].abs().mean()):.4f}")


if __name__ == "__main__":
    main()
