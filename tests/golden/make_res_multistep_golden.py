"""Node-level golden vectors of the res_multistep sampler from the REAL reference node layer (run in the build container only).

    python tests/golden/make_res_multistep_golden.py     # writes tests/golden/node_ksampler_res_multistep{,_mix}.npz

The same generator as `make_node_golden.py` -- the unmodified reference `nodes.py` over minicomfy, on the CPU, with
`torch.randn_like` on a recorded fp16-exact tape -- run on two more cases: `LanPaint_KSampler` with sampler
"res_multistep" (karras, 6 steps, N = 2), with the pointwise network and with `_node_cases.mixing_denoiser`.
Six steps take both of sample_res_multistep's updates: Euler on the first step and on the step to sigma = 0, the
second-order RES step in between.  The node's extra_args carry the seed, so the sampler's own draw (multiplied by
sigma_up = 0) comes from a private generator and leaves the tape alone.
"""
from __future__ import annotations

import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import make_node_golden as G  # noqa: E402

CASE = dict(name="node_ksampler_res_multistep", node="LanPaint_KSampler", shape=(1, 4, 8, 8), mask=(1, 1, 8, 8),
            args=dict(seed=7, steps=6, cfg=5.0, sampler_name="res_multistep", scheduler="karras", denoise=1.0,
                      LanPaint_NumSteps=2, LanPaint_PromptMode="Image First", Inpainting_mode=G.IMAGE_MODE))
CASES = [CASE, dict(CASE, name=CASE["name"] + "_mix", net="mixing")]


def main():
    G.CASES = CASES     # make_node_golden.main writes the cases of its module's list
    G.main(["--only", "^node_ksampler_res_multistep"])


if __name__ == "__main__":
    main()
