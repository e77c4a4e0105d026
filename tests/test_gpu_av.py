"""GPU: MiniMax-H3 AV per-row schedule (SURVEY 8f rank 4) against outputs of the REFERENCE engine called with
current_times_audio / audio_indicator / audio_correction (tests/golden/make_golden.py --av), plus the numeric
known answers of the reference's own tests/test_av_schedule.py, and against the oracle's AV path on the same torch
generator at sizes the fixtures cannot hold."""
import glob
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, load_golden
from _support import make_model, max_rel, synth_inputs
from oracle import langevin_oracle as O

pytestmark = pytest.mark.gpu
AV_CASES = sorted(os.path.splitext(os.path.basename(p))[0] for p in glob.glob(os.path.join(GOLDEN_DIR, "aux_av_*.npz")))


def _engine(model, n, lam=5.0, **kw):
    from lanpaint_b200.engine import LanPaint
    return LanPaint(model, NSteps=n, Friction=15.0, Lambda=lam, Beta=1.0, StepSize=0.2, IS_FLOW=True, MinStepFrac=1.0, **kw)


@pytest.mark.parametrize("name", AV_CASES)
def test_av_schedule_matches_reference(name, cuda_device):
    from lanpaint_b200.engine import NoiseTape
    assert len(AV_CASES) >= 4
    z = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    g = load_golden(name)
    meta = g["meta"]
    dev = cuda_device
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    x, y, noise = t(g["x"]), t(g["y"]), t(g["noise"])
    mask = t(z["mask"].astype(np.float32))
    sigma = t(g["sigma"])
    times = (t(g["ve"]), t(g["abt"]), t(g["flow_t"]))
    times_a = (t(z["ve_a"]), t(z["abt_a"]), t(z["flow_a"]))
    ai = torch.zeros((1, 1, x.shape[-1]), device=dev)
    ai[..., meta["video_n"]:] = 1.0
    corr = None if meta["corr"] is None else (1.0 - ai) + meta["corr"] * ai
    tape = NoiseTape([t(d) for d in g["tape"]])
    model = make_model("two_heads", True)
    eng = _engine(model, meta["n_steps"], rng=tape)
    out = eng(x, y, noise, sigma, mask, times, {}, 0, n_steps=meta["n_steps"], current_times_audio=times_a,
              audio_indicator=ai, audio_correction=corr)
    assert tape.pos == meta["n_draws"] and model.calls == meta["n_steps"] + 1
    assert max_rel(out, torch.from_numpy(g["out"])) <= 2e-5
    assert max_rel(x, torch.from_numpy(g["x_new"])) <= 2e-5


def test_replace_step_uses_audio_sigma_on_audio_rows(cuda_device):
    """reference tests/test_av_schedule.py:204-219."""
    dev = cuda_device
    x = torch.zeros(1, 1, 8, device=dev)
    y, noise = torch.zeros_like(x), torch.ones_like(x)
    ai = torch.zeros(1, 1, 8, device=dev)
    ai[..., 5:] = 1.0
    d = lambda v: torch.tensor([v], device=dev)
    model = make_model("identity", True)
    eng = _engine(model, 0, lam=1.0)
    eng.IS_FLOW = False
    eng(x, y, noise, d(0.5), torch.ones_like(x), (d(1.0), d(0.5), d(0.5)), None, 0, n_steps=0,
        current_times_audio=(d(0.25), d(0.9), d(0.2)), audio_indicator=ai)
    inp = model.last_input.flatten()
    assert inp[0].item() == pytest.approx(0.5) and inp[-1].item() == pytest.approx(0.2)


def test_non_suffix_indicator_is_rejected(cuda_device):
    dev = cuda_device
    x = torch.zeros(1, 1, 8, device=dev)
    ai = torch.zeros(1, 1, 8, device=dev)
    ai[..., 2:4] = 1.0
    d = lambda v: torch.tensor([v], device=dev)
    eng = _engine(make_model("identity", True), 1)
    with pytest.raises(NotImplementedError):
        eng(x, x.clone(), torch.ones_like(x), d(0.5), torch.ones_like(x), (d(1.0), d(0.5), d(0.5)), None, 0, n_steps=1,
            current_times_audio=(d(0.25), d(0.9), d(0.2)), audio_indicator=ai)


# (id, shape, split, correction, flow, n_steps, video sigma, audio sigma)
SAME_SEED_AV = [
    ("flow-5M-corr", (1, 1, 5_000_000), 2_500_000, 0.625, True, 3, 0.6, 0.3),
    ("flow-16lines-corr", (1, 16, 40960), 30720, 1.3, True, 4, 0.8, 0.5),
    ("odd-split", (1, 4, 4099), 3001, 0.8, True, 3, 0.7, 0.2),
    ("no-corr", (1, 4, 8192), 6144, None, True, 3, 0.6, 0.9),
    ("ve-corr", (1, 4, 8192), 5000, 0.625, False, 3, 1.5, 0.4),
    ("split-nlast", (1, 4, 8192), 8192, 1.3, True, 3, 0.6, 0.3),
    ("all-audio", (1, 4, 8192), 0, 1.3, True, 3, 0.6, 0.3),
]


@pytest.mark.parametrize("case", SAME_SEED_AV, ids=lambda c: c[0])
def test_av_same_seed_matches_oracle_on_gpu(case, cuda_device):
    """The engine's AV path against O.outer_step(..., audio=O.Audio(...)) on torch's global CUDA generator: the same
    draws in the same order, every position on its own schedule and correction.  The all-audio indicator is the
    case where the split starts at 0: every position is on the audio schedule."""
    from lanpaint_b200.engine import LanPaint
    _, shape, split, c, flow, n, s_v, s_a = case
    dev = cuda_device
    x, y, noise, m = synth_inputs(shape, seed=3, device=dev)
    mask = m.expand(shape).contiguous()
    sig, sig_a = torch.tensor([s_v], device=dev), torch.tensor([s_a], device=dev)
    times, times_a = O.times_from_sigma(sig, flow), O.times_from_sigma(sig_a, flow)
    ai = torch.zeros((1, 1, shape[-1]), device=dev)
    ai[..., split:] = 1.0
    corr = None if c is None else (1.0 - ai) + c * ai
    hp = O.Hyper(n_steps=n, min_step_frac=1.0, flow=flow)
    torch.manual_seed(1234)
    out_o, x_o = O.outer_step(make_model("two_heads", flow), x.clone(), y, noise, sig, mask, times, hp, n_steps=n,
                              audio=O.Audio(ai, times_a, corr))
    off_o = torch.cuda.default_generators[dev.index].get_offset()

    torch.manual_seed(1234)
    model = make_model("two_heads", flow)
    eng = LanPaint(model, NSteps=n, Friction=15.0, Lambda=5.0, Beta=1.0, StepSize=0.2, IS_FLOW=flow, MinStepFrac=1.0,
                   rng="torch")
    xe = x.clone()
    out_e = eng(xe, y, noise, sig, mask, tuple(times), {}, 0, n_steps=n, current_times_audio=tuple(times_a),
                audio_indicator=ai, audio_correction=corr)
    off_e = torch.cuda.default_generators[dev.index].get_offset()
    assert off_e == off_o, "the generator must advance exactly as the reference's randn_like calls do"
    assert model.calls == n + 1
    e_out, e_x = max_rel(out_e, out_o), max_rel(xe, x_o)
    assert e_out <= 2e-5 and e_x <= 2e-5, (e_out, e_x)
