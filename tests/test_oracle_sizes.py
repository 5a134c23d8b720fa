"""Images of another size than a net's image_size (non-square included), on the CPU.

The oracle (oracle/sr3_oracle.py) places attention by the construction-time resolution and runs everything else at the input's size, as the
reference does; it is pinned here to the unmodified reference's outputs in tests/golden/sr3_sizes_golden.pt (written by
tests/golden/make_sizes_golden.py from the cases and inputs of tests/_sizes_inputs.py).  The GPU tests (tests/test_gpu_sizes.py) compare
against the same fixture.  Also: the supported-size rule, in Python and in the library (which refuses before touching a device)."""
import ctypes
import os

import pytest
import torch

import _sizes_inputs as si
from oracle import sr3_oracle as orc

HERE = os.path.dirname(os.path.abspath(__file__))


def cfg_of(name):
    unet, image_size = si.CASES[name][:2]
    return orc.UNetConfig(unet["in_channel"], unet["out_channel"], unet["inner_channel"], 32, tuple(unet["channel_multiplier"]),
                          tuple(unet["attn_res"]), unet["res_blocks"], 0.0, image_size)


@pytest.fixture(scope="module")
def sizes():
    return torch.load(os.path.join(HERE, "golden", "sr3_sizes_golden.pt"), map_location="cpu", weights_only=False)


def rel(a, b):
    return ((a - b).norm() / b.norm()).item()


@pytest.mark.timeout(900)
@pytest.mark.parametrize("name", sorted(si.CASES))
def test_oracle_matches_reference_at_other_sizes(sizes, name):
    g, cfg, inp = sizes[name], cfg_of(name), si.inputs(name)
    sd = orc.init_state_dict(cfg, g["seed"])
    taps = {}
    with torch.no_grad():
        eps = orc.unet_forward(sd, cfg, inp["x"], inp["noise_level"], taps)
    assert eps.shape == inp["x"][:, :3].shape
    assert rel(si.eps_crop(name, eps), g["eps"]) < 5e-6
    assert sorted(g["taps"]) == sorted(si.CASES[name][7])
    for layer, ref in g["taps"].items():
        assert rel(si.tap_crop(name, layer, taps[layer]), ref) < 5e-6, layer


@pytest.mark.timeout(1800)
def test_oracle_pmv_and_loop_at_128x256(sizes):
    name = si.LOOP_CASE
    g, cfg, inp = sizes[name], cfg_of(name), si.inputs(name)
    sd = orc.init_state_dict(cfg, g["seed"])
    sch = orc.make_schedule(si.SCHED)
    b = inp["x_t"].shape[0]
    with torch.no_grad():
        for t in si.T_EVAL:
            nl = orc.noise_level_for_t(sch, t, b)
            e = orc.unet_forward(sd, cfg, torch.cat([inp["cond"], inp["x_t"]], 1), nl)
            assert rel(si.eps_crop(name, e), g["eps_t"][t]) < 5e-6, t
            m, lv = orc.p_mean_variance(sd, cfg, sch, inp["x_t"], t, True, inp["cond"])
            assert rel(si.eps_crop(name, m), g["pmv"][t][0]) < 5e-6 and float(lv) == float(g["pmv"][t][1]), t
        d = si.loop_inputs()
        loop = orc.p_sample_loop(sd, cfg, orc.make_schedule(si.SCHED10), inp["cond"], d["x_T"], list(d["noises"]), True, continous=True)
    assert loop.shape == (b * 11, 3, 128, 256)
    assert rel(si.eps_crop(name, loop[5 * b:6 * b]), g["loop_mid"]) < 2e-5
    assert rel(si.eps_crop(name, loop[-b:]), g["loop_last"]) < 2e-5


# (levels, height, width) -> lowest level, or the part of the message naming the rule
ACCEPTED = [(5, 128, 128, (8, 8)), (5, 128, 256, (8, 16)), (5, 256, 128, (16, 8)), (5, 512, 512, (32, 32)), (5, 64, 64, (4, 4)),
            (2, 32, 64, (16, 32)), (3, 16, 16, (4, 4)), (1, 8, 8, (8, 8)), (1, 8, 64, (8, 64)), (4, 64, 1024, (8, 128))]
REFUSED = [(4, 16, 16, "< 4"), (5, 32, 64, "< 4"), (5, 64, 128, "lowest UNet level 4x8"), (3, 16, 32, "lowest UNet level 4x8"),
           (1, 8, 4, "lowest UNet level 8x4"), (5, 96, 128, "powers of two"), (2, 32, 48, "powers of two"), (5, 0, 128, "positive")]


@pytest.mark.parametrize("levels,h,w,lowest", ACCEPTED)
def test_size_rule_accepts(levels, h, w, lowest):
    from sr3_b200 import _native
    assert _native.check_image_size(levels, h, w) == lowest


@pytest.mark.parametrize("levels,h,w,msg", REFUSED)
def test_size_rule_refuses(levels, h, w, msg):
    from sr3_b200 import _native
    with pytest.raises(_native.UnsupportedSizeError, match=msg) as e:
        _native.check_image_size(levels, h, w)
    assert f"{h}x{w}" in str(e.value)
    assert isinstance(e.value, ValueError) and isinstance(e.value, RuntimeError)


@pytest.mark.parametrize("levels,h,w,msg", REFUSED)
def test_library_refuses_the_same_sizes_before_touching_a_device(levels, h, w, msg):
    """sr3_engine_create_sized applies the same rule first: it fails with the same message on a machine without a GPU too."""
    from sr3_b200 import _native
    c = _native.UNetConfigC()
    c.in_channel, c.out_channel, c.inner_channel, c.norm_groups, c.n_mults = 6, 3, 64, 32, levels
    for i in range(levels):
        c.channel_mults[i] = 1
    c.res_blocks, c.image_size, c.channels, c.conditional = 1, 16, 3, 1
    h_ = ctypes.c_void_p()
    assert _native.lib().sr3_engine_create_sized(ctypes.byref(c), 1, h, w, 0, ctypes.byref(h_)) != 0
    err = _native.lib().sr3_last_error().decode()
    assert msg in err and f"{h}x{w}" in err, err
    assert not h_.value


def test_sized_entry_point_is_exported():
    from sr3_b200 import _native
    assert "sr3_engine_create_sized" in _native.EXPORTED_SYMBOLS
    assert hasattr(ctypes.CDLL(_native.LIB_PATH), "sr3_engine_create_sized")
