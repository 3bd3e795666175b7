"""CPU: oracle/sweep_oracle.py reproduces, bit for bit, every array the unmodified reference wrote in
tests/golden/sweep_ref.npz (Simulator.render's PNGs, clouds and video frames, Trainer.test's PNGs / video frames and
clouds, the validation panels), so the GPU tests can hold the CUDA op to the oracle on frames the reference never saw."""
import os

import numpy as np
import pytest

import sweep_cases as SC
from oracle import sweep_oracle as SO

FX = np.load(os.path.join(os.path.dirname(__file__), "golden", "sweep_ref.npz"), allow_pickle=False)
LUT_I, LUT_D = FX["lut_intensity"], FX["lut_depth"]


@pytest.mark.parametrize("case", sorted(SC.SIM))
def test_simulator_outputs(case):
    refine, fov = SC.SIM[case]
    fr = SC.frames(FX, case)
    n = FX[f"sim_{case}_times"].shape[0]
    for i in range(n):
        f = fr[i]
        panel, _, _, cloud = SO.sim(SC.raydrop_of(f, refine), f["image"][..., 1], f["depth"], SC.SCALE, fov, LUT_I, LUT_D)
        assert SC.same(FX, f"sim_{case}_png{i}", panel)
        assert SC.same(FX, f"sim_{case}_video{i}", panel[..., ::-1])
        assert SC.same(FX, f"sim_{case}_npy{i}", cloud)


@pytest.mark.parametrize("case", sorted(SC.TEST))
def test_trainer_test_outputs(case):
    alpha_r, refine, _ = SC.TEST[case]
    for i, f in enumerate(SC.frames(FX, case)):
        raydrop, inten, depth, _, points = SO.test(SC.raydrop_of(f, refine), f["image"][..., 1], f["depth"], SC.SCALE,
                                                   alpha_r, (2.0, 26.9), LUT_I, LUT_D)
        if f"test_{case}_raydrop{i}" in FX.files:
            assert SC.same(FX, f"test_{case}_raydrop{i}", raydrop)
        assert SC.same(FX, f"test_{case}_intensity{i}", inten)
        assert SC.same(FX, f"test_{case}_depth{i}", depth)
        assert SC.same(FX, f"test_{case}_points{i}", points)


@pytest.mark.parametrize("case", SC.EVAL)
def test_validation_panel(case):
    for i, f in enumerate(SC.frames(FX, case)):
        panel = SO.evaluate(f["unet"], f["image"][..., 1], f["depth"], LUT_I, LUT_D)
        assert SC.same(FX, f"eval_{case}_png{i}", panel)


def test_cases_reach_the_edges():
    """The frames hold what the rules are about: wrapped depths, NaN, exact 0.5 ray drops and float16 maps."""
    f = SC.frames(FX, "66x1030_f16")[0]
    assert f["unet"].dtype == np.float16 and (f["unet"] == np.float16(0.5)).any()
    assert (f["depth"] * 255 >= 256).any() and np.isnan(f["depth"]).any() and np.isnan(f["image"]).any()
    assert FX["sim_32x1024_origins"].shape == (1, 3) and FX["sim_66x1030_origins"].shape == (2, 3)
