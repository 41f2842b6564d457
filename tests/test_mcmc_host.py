"""CPU: the host side of the MCMC strategy -- the C ABI's argument checks (no kernel runs), the refinement schedule,
the Gaussian-count trajectory under the cap, the configuration's checks and GaussianModel's refusal of it."""
import ctypes as C
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mcmc_f64 as ref  # noqa: E402

from opensplat_b200 import capi  # noqa: E402
from opensplat_b200.mcmc import MCMCConfig, grow_count, refines, seed_key  # noqa: E402

P = C.c_void_p(256)      # any 256-byte aligned address: every call below is rejected before it is used
BAD = -1


def _segs(*rows):
    return (capi.RowSegment * len(rows))(*[capi.RowSegment(64 * i, r, 0) for i, r in enumerate(rows)])


def test_capi_mcmc_argument_checks():
    L = capi.lib()
    assert L.gsb_mcmc_workspace_bytes(-1) == 0
    sizes = [L.gsb_mcmc_workspace_bytes(n) for n in (1, 4096, 4097, 1 << 20, 5 << 20)]
    assert sizes == sorted(sizes) and sizes[0] > 0
    ws = L.gsb_mcmc_workspace_bytes(1000)
    # plan: negative or too large n, no result, misaligned or short workspace, dead flags without an output
    assert L.gsb_mcmc_plan(-1, P, 0.005, 1, P, ws, P, P, P, None) == BAD
    assert L.gsb_mcmc_plan(1 << 29, P, 0.005, 1, P, 1 << 40, P, P, P, None) == BAD
    assert L.gsb_mcmc_plan(1000, P, 0.005, 1, P, ws, P, P, None, None) == BAD
    assert L.gsb_mcmc_plan(1000, P, 0.005, 1, C.c_void_p(272), ws, P, P, P, None) == BAD
    assert L.gsb_mcmc_plan(1000, P, 0.005, 1, P, ws - 1, P, P, P, None) == BAD
    assert L.gsb_mcmc_plan(1000, P, 0.005, 1, P, ws, P, None, P, None) == BAD
    # sample: negative counts, draws from an empty set, missing outputs; nothing to do is a no-op
    assert L.gsb_mcmc_sample(-1, 10, P, 0, 0, 1, 1, P, P, None) == BAD
    assert L.gsb_mcmc_sample(5, 0, P, 0, 0, 1, 1, P, P, None) == BAD
    assert L.gsb_mcmc_sample(5, 10, P, 0, 0, 1, 1, None, P, None) == BAD
    assert L.gsb_mcmc_sample(0, 0, None, 0, 0, 1, 1, None, None, None) == 0
    # relocate / copy_rows: the segment table (count, row length), missing moments when they are to be zeroed
    assert L.gsb_mcmc_relocate(10, P, 0.005, P, P, 0, 9, _segs(*[3] * 9), P, P, None) == BAD
    assert L.gsb_mcmc_relocate(10, P, 0.005, P, P, 0, 2, _segs(3, 0), P, P, None) == BAD
    assert L.gsb_mcmc_relocate(10, P, 0.005, P, P, 1, 2, _segs(3, 4), None, P, None) == BAD
    assert L.gsb_mcmc_relocate(10, P, 0.005, P, P, 0, 1, None, P, P, None) == BAD
    assert L.gsb_mcmc_relocate(0, None, 0.005, None, None, 0, 1, _segs(3), None, None, None) == 0
    assert L.gsb_mcmc_copy_rows(-1, P, P, 1, _segs(3), P, None) == BAD
    assert L.gsb_mcmc_copy_rows(4, None, P, 1, _segs(3), P, None) == BAD
    assert L.gsb_mcmc_copy_rows(0, None, None, 1, _segs(3), None, None) == 0
    # regularize / add_noise / draws
    assert L.gsb_mcmc_regularize(-1, P, P, 0.1, 0.1, P, P, None) == BAD
    assert L.gsb_mcmc_regularize(10, P, P, 0.1, 0.1, None, P, None) == BAD
    assert L.gsb_mcmc_add_noise(-1, P, P, P, 0, 0, 1, 1.0, P, None) == BAD
    assert L.gsb_mcmc_add_noise(10, P, P, C.c_void_p(260), 0, 0, 1, 1.0, P, None) == BAD
    assert L.gsb_mcmc_draws(-1, 0, 0, 1, 0, P, P, None) == BAD
    assert L.gsb_mcmc_draws(10, 0, 0, 1, 0, C.c_void_p(260), None, None) == BAD
    assert L.gsb_mcmc_draws(10, 0, 0, 1, 0, None, None, None) == BAD
    assert L.gsb_mcmc_draws(0, 0, 0, 1, 0, None, None, None) == 0


def test_schedule():
    c = MCMCConfig()
    steps = [s for s in range(1, 30001) if refines(c, s)]
    assert steps[0] == 600 and steps[-1] == 24900 and len(steps) == 244
    assert all(refines(c, s) == ref.refines(s) for s in range(1, 30001))
    assert not refines(c, 500) and not refines(c, 25000) and not refines(c, 650)
    c = MCMCConfig(refine_start=0, refine_stop=10, refine_every=3)
    assert [s for s in range(1, 20) if refines(c, s)] == [3, 6, 9]


@pytest.mark.parametrize("n0,cap", [(1000, 1_000_000), (100_000, 150_000), (7, 10), (20, 20), (0, 100),
                                    (5000, 4000)])
def test_count_trajectory(n0, cap):
    n, traj = n0, [n0]
    for _ in range(300):
        n += grow_count(n, cap)
        traj.append(n)
    want = [n0]
    for _ in range(300):
        want.append(max(want[-1], min(cap, int(1.05 * want[-1]))))
    assert traj == want
    assert all(b >= a for a, b in zip(traj, traj[1:]))
    if n0 <= cap:
        assert max(traj) <= cap
    else:                                     # a set above the cap neither grows nor shrinks
        assert traj == [n0] * 301
    assert grow_count(n0, cap) == ref.grow_count(n0, cap)
    if n0 >= 20 and cap >= n0 * 2:            # 5 % per refinement while below the cap
        assert traj[1] == int(1.05 * n0)


def test_config_checks_and_seed_key():
    for bad in (dict(min_opacity=0.0), dict(min_opacity=1.0), dict(refine_every=0), dict(cap_max=-1),
                dict(noise_lr=-1.0), dict(opacity_reg=-0.1), dict(seed=-1), dict(seed=1 << 64)):
        with pytest.raises(ValueError):
            MCMCConfig(**bad)
    s = 0x0123456789abcdef
    assert seed_key(s) == ref.seed_key(s) == (0x89abcdef, 0x01234567)
    assert MCMCConfig().seed == 0 and MCMCConfig().cap_max == 1_000_000 and MCMCConfig().max_steps == 30_000


def test_gaussian_model_refuses_the_mcmc_config():
    from opensplat_b200.model import GaussianModel
    with pytest.raises(ValueError):
        GaussianModel({}, MCMCConfig(), device="cpu")
