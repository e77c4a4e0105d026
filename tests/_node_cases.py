"""Shared by tests/golden/make_node_golden.py (which drives the REFERENCE's node layer) and the node-level
parity tests (which drive lanpaint_b200's): how a case's JSON arguments become the positional call ComfyUI's
executor makes.  Test infrastructure."""
import torch

import minicomfy

IMAGE_MODE = "🖼️ Image Inpainting"
VIDEO_MODE = "🎬 Video Inpainting"


def denoiser(x, sigma, cond):
    """pointwise cond-dependent x0 prediction; `cond` is a float standing in for CONDITIONING"""
    return 0.7 * x + 0.1 * torch.tanh(x) + cond


def mixing_denoiser(x, sigma, cond):
    """`denoiser` plus a fixed coupling of every element to its neighbours over channels and every spatial /
    sequence axis (never the batch axis: requests stay independent).  With a pointwise network a free element's
    trajectory never reads a known one, so nothing a job does at known positions reaches the final latent except the
    paste `out = y`; with this one the known region feeds the free region through every model call.  Elementwise
    ops and `roll` only: no TF32, the same on CPU and GPU up to a tanh ulp, capturable in a CUDA graph."""
    out = 0.6 * x + 0.1 * torch.tanh(x) + cond
    for d in range(1, x.ndim):
        out = out + 0.05 * torch.roll(x, 1, d)
    return out


NETS = {"pointwise": denoiser, "mixing": mixing_denoiser}


def net_of(c):
    """The test network a case (a fixture's meta) was generated with."""
    return NETS[c.get("net", "pointwise")]


class FixedNoise:
    """a NOISE object for LanPaint_SamplerCustomAdvanced (ComfyUI's RandomNoise protocol: .seed, .generate_noise)"""

    def __init__(self, seed, image):
        self.seed, self.image = seed, image

    def generate_noise(self, latent):
        return self.image


POS, NEG = 0.3, -0.2


def build_patcher(c, device="cpu", net=None):
    """`net` (a counting wrapper, say) defaults to the case's own network, `net_of(c)`."""
    if net is None:
        net = net_of(c)
    mtype = getattr(minicomfy.ModelType, c.get("model_type", "EPS"))
    cls = minicomfy.WAN22 if c.get("wan22") else minicomfy.BaseModel
    base = cls(net, model_type=mtype, latent_channels=c["shape"][1], shift=c.get("shift", 1.0))
    return minicomfy.ModelPatcher(base, device)


def call_node(N, c, patcher, latent, noise_image=None):
    """The same positional call ComfyUI's executor makes, on node module `N` (the reference's or lanpaint_b200's)."""
    a = c["args"]
    if c["node"] == "outer_sample_av_pack":
        return call_av_pack(N, c, patcher, latent, noise_image)
    node = N.NODE_CLASS_MAPPINGS[c["node"]]()
    if c["node"] == "LanPaint_KSampler":
        return node.sample(patcher, a["seed"], a["steps"], a["cfg"], a["sampler_name"], a["scheduler"], POS, NEG, latent,
                           a["denoise"], a["LanPaint_NumSteps"], a["LanPaint_PromptMode"], "", a["Inpainting_mode"])
    if c["node"] == "LanPaint_KSamplerAdvanced":
        return node.sample(patcher, a["add_noise"], a["noise_seed"], a["steps"], a["cfg"], a["sampler_name"],
                           a["scheduler"], POS, NEG, latent, a["start_at_step"], a["end_at_step"],
                           a["return_with_leftover_noise"], a["LanPaint_NumSteps"], a["LanPaint_Lambda"],
                           a["LanPaint_StepSize"], a["LanPaint_PromptMode"], "", a["Inpainting_mode"])
    kind, n = a["sigmas"]
    sig = minicomfy.get_sigmas_karras(n, 0.0292, 14.6146)
    sampler = minicomfy.ksampler(a["sampler"])
    if c["node"] == "LanPaint_SamplerCustom":
        return node.sample(patcher, sampler, sig, a["add_noise"], a["noise_seed"], a["cfg"], POS, NEG, latent,
                           a["LanPaint_NumSteps"], a["LanPaint_PromptMode"], "")
    guider = minicomfy.CFGGuider(patcher)
    guider.set_conds(POS, NEG)
    guider.set_cfg(a["cfg"])
    return node.sample(FixedNoise(a["noise_seed"], noise_image), guider, sampler, sig, latent, a["LanPaint_NumSteps"],
                       a["LanPaint_Lambda"], a["LanPaint_StepSize"], a["LanPaint_PromptMode"], "")


# ---- MiniMax-H3 AV flat pack (nodes.py:188-191, 254-275, 340-349) -----------------------------------------------
# comfy.ldm.minimax.model is not in this sandbox (ComfyUI is absent): these stand-ins are patched into BOTH node
# modules as `time_shift_sigma` / `time_shift_slope`; the parity statement is about what the node layers do with them.
def av_shift_sigma(s, sv, sa):
    return sa * s / (sv + (sa - sv) * s)


def av_shift_slope(s, sv, sa):
    return sa * sv / (sv + (sa - sv) * s) ** 2


def call_av_pack(N, c, patcher, latent, noise_image):
    """A nested (video, audio) latent arrives at the patched CFGGuider.outer_sample as one flat pack plus
    `latent_shapes`; ComfyUI's CFGGuider.sample does that unpacking, so the seam itself is called here."""
    a = c["args"]
    N._LanPaint_test_shift = (N.time_shift_sigma, N.time_shift_slope)
    N.time_shift_sigma, N.time_shift_slope = av_shift_sigma, av_shift_slope
    try:
        net = patcher.model.diffusion_model
        net.sigma_shift_video, net.sigma_shift_audio = a["shift_video"], a["shift_audio"]
        patcher.LanPaint_StepSize, patcher.LanPaint_Lambda, patcher.LanPaint_Beta = 0.2, 5.0, 1.0
        patcher.LanPaint_NumSteps, patcher.LanPaint_MinStepFrac, patcher.LanPaint_Friction = a["LanPaint_NumSteps"], 1.0, 15.0
        patcher.LanPaint_EarlyStop, patcher.LanPaint_InnerThreshold, patcher.LanPaint_InnerPatience = 1, 0.0, 1
        patcher.LanPaint_cfg_BIG = a["cfg"]
        guider = minicomfy.CFGGuider(patcher)
        guider.set_conds(POS, NEG)
        guider.set_cfg(a["cfg"])
        sig = torch.tensor(a["sigmas"], dtype=torch.float32)
        with N.override_sample_function():
            out = type(guider).outer_sample(guider, noise_image, latent["samples"], minicomfy.ksampler("euler"), sig,
                                            denoise_mask=latent["noise_mask"], seed=a["seed"],
                                            latent_shapes=[(1, a["n_video"]), (1, a["n_audio"])])
        return ({"samples": out.cpu(), "noise_mask": latent["noise_mask"]},)
    finally:
        N.time_shift_sigma, N.time_shift_slope = N._LanPaint_test_shift
        del N._LanPaint_test_shift
