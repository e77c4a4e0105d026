"""Node-level golden vectors of the dpm_2 sampler from the REAL reference node layer (run in the build container only).

    python tests/golden/make_dpm_2_golden.py     # writes tests/golden/node_ksampler_dpm_2{,_mix}.npz

The same generator as `make_node_golden.py` -- the unmodified reference `nodes.py` over minicomfy, on the CPU, with
`torch.randn_like` on a recorded fp16-exact tape -- run on two more cases: `LanPaint_KSampler` with sampler "dpm_2"
(karras, 5 steps, N = 2), with the pointwise network and with `_node_cases.mixing_denoiser`.  KSampler drops dpm_2's
penultimate sigma, and the reference's per-sigma wrapper runs at every midpoint sigma the sampler asks for, so these
fixtures pin the wrapper at sigmas outside the schedule (n_eff by its nearest-sigma rule).
"""
from __future__ import annotations

import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import make_node_golden as G  # noqa: E402

DPM_2 = dict(name="node_ksampler_dpm_2", node="LanPaint_KSampler", shape=(1, 4, 8, 8), mask=(1, 1, 8, 8),
             args=dict(seed=6, steps=5, cfg=5.0, sampler_name="dpm_2", scheduler="karras", denoise=1.0,
                       LanPaint_NumSteps=2, LanPaint_PromptMode="Image First", Inpainting_mode=G.IMAGE_MODE))
CASES = [DPM_2, dict(DPM_2, name=DPM_2["name"] + "_mix", net="mixing")]


def main():
    G.CASES = CASES     # make_node_golden.main writes the cases of its module's list
    G.main(["--only", "^node_ksampler_dpm_2"])


if __name__ == "__main__":
    main()
