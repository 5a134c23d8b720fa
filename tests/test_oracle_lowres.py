"""Pins oracle/sr3_oracle.py to the unmodified reference for UNets whose lowest level is 4x4 (tests/golden/sr3_lowres_golden.pt, written by
tests/golden/make_lowres_golden.py from the inputs of tests/_lowres_inputs.py): a 16 -> 8 -> 4 net with its middle attention at 4x4, an
unconditional 32 -> 4 net and the 16->64 config.  The GPU tests of these nets (tests/test_gpu_lowres.py) compare against the same fixture."""
import os

import numpy as np
import pytest
import torch

import _lowres_inputs as li
from oracle import sr3_oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))
TINY4 = orc.UNetConfig(6, 3, 64, 32, (1, 2, 2), (), 1, 0.0, 16)
UNCOND32 = orc.UNetConfig(3, 3, 64, 32, (1, 2, 4, 8), (), 1, 0.0, 32)
SR16_64 = orc.UNetConfig(6, 3, 64, 32, (1, 2, 4, 8, 8), (16,), 2, 0.0, 64)


@pytest.fixture(scope="module")
def lowres():
    return torch.load(os.path.join(HERE, "golden", "sr3_lowres_golden.pt"), map_location="cpu", weights_only=False)


def rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def test_tiny_4x4_net_layers_eps_and_pmv(lowres):
    g, inp = lowres["tiny4"], li.tiny4()
    sd = orc.init_state_dict(TINY4, g["seed"])
    sch = orc.make_schedule(li.SCHED)
    taps = {}
    with torch.no_grad():
        eps = orc.unet_forward(sd, TINY4, inp["x"], inp["noise_level"], taps)
        assert rel(eps, g["eps"]) < 2e-6
        for k, v in g["taps"].items():
            assert rel(taps[k][:1], v) < 2e-6, k
        for t, e in g["eps_t"].items():
            nl = orc.noise_level_for_t(sch, t, e.shape[0])
            assert rel(orc.unet_forward(sd, TINY4, torch.cat([inp["cond"], inp["x_t"]], 1), nl), e) < 2e-6, t
            m, lv = g["pmv"][t]
            om, olv = orc.p_mean_variance(sd, TINY4, sch, inp["x_t"], t, True, inp["cond"])
            assert rel(om, m) < 5e-6 and float(olv) == float(lv), t


def test_tiny_4x4_loop_and_losses(lowres):
    g, inp, d = lowres["tiny4_diffusion"], li.tiny4(), li.tiny4_diffusion()
    sd = orc.init_state_dict(TINY4, 0)
    sch = orc.make_schedule(li.SCHED10)
    with torch.no_grad():
        loop = orc.p_sample_loop(sd, TINY4, sch, inp["cond"], d["x_T"], list(d["noises"]), True, continous=True)
        assert loop.shape == (3 * 11, 3, 16, 16)
        assert rel(loop[15:18], g["loop_mid"]) < 2e-5 and rel(loop[-3:], g["loop_last"]) < 2e-5
        _, gamma = orc.draw_gamma(sch, 3, np.random.RandomState(d["np_seed"]))
        loss = orc.p_losses(sd, TINY4, sch, d["hr"], inp["cond"], gamma, d["noise"])
    assert abs(loss.item() - g["loss"].item()) / g["loss"].item() < 1e-5


def test_unconditional_32_net(lowres):
    g = lowres["uncond32"]
    x_t = li.uncond32()["x_t"]
    sd = orc.init_state_dict(UNCOND32, g["seed"])
    sch = orc.make_schedule(li.SCHED)
    with torch.no_grad():
        for t, e in g["eps"].items():
            assert rel(orc.unet_forward(sd, UNCOND32, x_t, orc.noise_level_for_t(sch, t, e.shape[0])), e) < 2e-6


@pytest.mark.timeout(600)
def test_16_64_config(lowres):
    g, s = lowres["sr16_64"], li.sr16_64()
    sd = orc.init_state_dict(SR16_64, g["seed"])
    sch = orc.make_schedule(li.SCHED)
    with torch.no_grad():
        for t, e in g["eps"].items():
            nl = orc.noise_level_for_t(sch, t, e.shape[0])
            assert rel(orc.unet_forward(sd, SR16_64, torch.cat([s["cond"], s["x_t"]], 1), nl)[li.CROP], e) < 2e-6, t
            m, lv = g["pmv"][t]
            om, olv = orc.p_mean_variance(sd, SR16_64, sch, s["x_t"], t, True, s["cond"])
            assert rel(om[li.CROP], m) < 5e-6 and float(olv) == float(lv), t
