"""GPU: the 3DGS-MCMC strategy (DESIGN.md D20) -- csrc/mcmc.cu against the float64 restatement tests/mcmc_f64.py
(Philox words bit-exact, normals within 2e-6, sample indices exact except within a certified scan bound, counts
exact, relocated logits / log-scales within 1 ulp, copied rows and moments bit-exact, regulariser and noise within
bounds derived from their fp32 operation counts), the edge cases, and SplatTrainer(cfg=MCMCConfig): equal to a plain
trainer with MCMCRefiner.finish_step after each step, the regulariser's exact share of the gradient, seeded
determinism, a 1500-step run under the cap, several views per step, the anti-aliased mode and data-parallel replicas
(tools/check_parallel_trainer.py --mcmc)."""
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import mcmc_f64 as ref  # noqa: E402

from opensplat_b200 import capi  # noqa: E402
from opensplat_b200.mcmc import MCMCConfig, MCMCRefiner, grow_count  # noqa: E402
from opensplat_b200.parallel import flat_layout, flat_views  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24                      # fp32 unit roundoff


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def dev_sigmoid(logits):
    """The fp32 opacities 1.f / (1.f + expf(-logit)) as the device forms them (gsb_activate_forward)."""
    lg = cu(np.asarray(logits, np.float32).reshape(-1))
    n = lg.numel()
    if n == 0:
        return np.zeros(0, np.float32)
    z3, z4 = torch.zeros((n, 3), device=DEV), torch.ones((n, 4), device=DEV)
    out = [torch.empty((n, k), device=DEV) for k in (3, 4, 1, 3)]
    capi.check(capi.lib().gsb_activate_forward(n, capi.ptr(z3), capi.ptr(z3), capi.ptr(z4), capi.ptr(lg),
                                               capi.ptr(torch.zeros(3, device=DEV)), *[capi.ptr(t) for t in out],
                                               capi.stream()))
    return out[2].reshape(-1).cpu().numpy()


def ulps(a, b):
    """|a - b| in units of the fp32 spacing at max(|a|, |b|)."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    sp = np.spacing(np.maximum(np.abs(a), np.abs(b)))
    return np.abs(a.astype(np.float64) - b.astype(np.float64)) / sp.astype(np.float64)


# ---- Philox -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed,step,tag", [(0, 1, 0), (0x0123456789abcdef, 600, 1), ((1 << 64) - 1, 29999, 2)])
def test_philox_words_and_normals(seed, step, tag):
    count = 200_003
    words = torch.empty((count, 4), dtype=torch.int32, device=DEV)
    z = torch.empty((count, 3), dtype=torch.float32, device=DEV)
    capi.check(capi.lib().gsb_mcmc_draws(count, seed & 0xffffffff, seed >> 32, step, tag, capi.ptr(words),
                                         capi.ptr(z), capi.stream()))
    want = ref.draws(count, seed, step, tag)
    assert np.array_equal(words.cpu().numpy().view(np.uint32).astype(np.uint64), want)
    assert np.abs(z.cpu().numpy() - ref.normals(want)).max() <= 2e-6


# ---- planning and sampling --------------------------------------------------------------------------------------

def _plan(logits, min_opacity, mask_dead):
    L, n = capi.lib(), len(logits)
    lg = cu(np.asarray(logits, np.float32))
    ws = torch.empty(max(L.gsb_mcmc_workspace_bytes(n), 1), dtype=torch.uint8, device=DEV)
    cdf = torch.empty(max(n, 1), dtype=torch.float64, device=DEV)
    dead = torch.full((max(n, 1),), -7, dtype=torch.int32, device=DEV)
    res = torch.full((4,), -7, dtype=torch.int32, device=DEV)
    capi.check(L.gsb_mcmc_plan(n, capi.ptr(lg), min_opacity, int(mask_dead), capi.ptr(ws), ws.numel(), capi.ptr(cdf),
                               capi.ptr(dead), capi.ptr(res), capi.stream()))
    return cdf, dead, res.cpu().tolist()


def _sample(cdf, n, m, seed, step, tag):
    samples = torch.empty(max(m, 1), dtype=torch.int32, device=DEV)
    counts = torch.full((n,), -7, dtype=torch.int32, device=DEV)
    capi.check(capi.lib().gsb_mcmc_sample(m, n, capi.ptr(cdf), seed & 0xffffffff, seed >> 32, step, tag,
                                          capi.ptr(samples), capi.ptr(counts), capi.stream()))
    return samples[:m].cpu().numpy(), counts.cpu().numpy()


def check_samples(got, cdf_dev, cdf_ref, u):
    """Sample indices exact, except where u T falls within the certified scan bound of the boundary between the
    device's index and the restatement's: there the neighbour is accepted.  Returns the number of such draws."""
    want = ref.sample(cdf_ref, u)
    bad = np.nonzero(got != want)[0]
    bound = ref.scan_bound(cdf_ref) + abs(float(cdf_dev[-1]) - float(cdf_ref[-1]))
    for j in bad:
        assert abs(int(got[j]) - int(want[j])) == 1, (j, got[j], want[j])
        edge = cdf_ref[min(got[j], want[j])]
        assert abs(u[j] * cdf_ref[-1] - edge) <= bound, (j, u[j] * cdf_ref[-1] - edge, bound)
    return len(bad)


@pytest.mark.parametrize("n,dead_frac", [(1, 0.0), (1000, 0.3), (4096, 0.5), (4097, 0.1), (300_001, 0.2),
                                         (1_100_000, 0.05)])
def test_plan_and_samples_against_the_restatement(n, dead_frac):
    rng = np.random.default_rng(n)
    logits = rng.uniform(-4, 4, n).astype(np.float32)
    logits[rng.uniform(size=n) < dead_frac] = -7.0       # o ~ 9e-4: dead
    o = dev_sigmoid(logits)
    for mask_dead in (True, False):
        cdf, dead, res = _plan(logits, 0.005, mask_dead)
        c = cdf.cpu().numpy()[:n]
        w = ref.weights(o, 0.005 if mask_dead else None)
        cref = np.cumsum(w)
        want_dead = np.nonzero(o <= np.float32(0.005))[0] if mask_dead else np.zeros(0, int)
        assert res == [len(want_dead), int(cref[-1] > 0), int((o > 0).any()), 0]
        assert np.array_equal(dead.cpu().numpy()[:len(want_dead)], want_dead)
        assert (np.diff(c) >= 0).all()                              # monotone
        assert np.abs(c - cref).max() <= ref.scan_bound(cref)
        assert (c[w == 0] == np.concatenate([[0.0], c])[:-1][w == 0]).all()   # a zero weight adds nothing
        if cref[-1] == 0:
            continue
        m = max(len(want_dead), 5000)
        tag = ref.RELOCATE_TAG if mask_dead else ref.GROW_TAG
        got, counts = _sample(cdf, n, m, 77, 600, tag)
        u = ref.uniform(*ref.draws(m, 77, 600, tag)[:, :2].T)
        check_samples(got, c, cref, u)
        assert (w[got] > 0).all()
        assert np.array_equal(counts, np.bincount(got, minlength=n))


# ---- the refinement on a pipeline's flat buffers ------------------------------------------------------------------

NAMES = ("means", "scales", "quats", "opacities", "coeffs")


def make_pipe(n, K=4, seed=0, logits=None):
    """A stand-in for SplatPipeline's Gaussian buffers (what MCMCRefiner reads): flat parameters and moments."""
    rng = np.random.default_rng(seed)
    offs, numel = flat_layout(n, K)
    pf = torch.zeros(numel, device=DEV)
    p = flat_views(pf, offs)
    host = {"means": rng.standard_normal((n, 3)), "scales": rng.uniform(-5, -1, (n, 3)),
            "quats": rng.standard_normal((n, 4)), "opacities": rng.uniform(-3, 3, (n, 1)),
            "coeffs": rng.standard_normal((n, K, 3))}
    if logits is not None:
        host["opacities"] = np.asarray(logits, np.float64).reshape(n, 1)
    for k in NAMES:
        p[k].copy_(cu(host[k].astype(np.float32)))
    m = torch.from_numpy(rng.standard_normal(numel).astype(np.float32)).to(DEV)
    v = torch.from_numpy(rng.uniform(0, 1, numel).astype(np.float32)).to(DEV)
    return SimpleNamespace(n=n, offs=offs, param_flat=pf, p=p, adam_m=m, adam_v=v)


def host_state(pipe):
    def d(flat):
        return {k: t.cpu().numpy().copy() for k, t in flat_views(flat, pipe.offs).items()}
    return d(pipe.param_flat), d(pipe.adam_m), d(pipe.adam_v)


def to_np(dct):
    return {k: t.detach().cpu().numpy() for k, t in dct.items()}


def check_update(got_p, want_p, rows):
    """Logits and log-scales of the updated rows within 1 ulp; everything else bit-exact."""
    for k in NAMES:
        g, w = got_p[k], want_p[k]
        assert g.shape == w.shape, k
        if k in ("opacities", "scales"):
            assert ulps(g[rows], w[rows]).max() <= 1.0, (k, ulps(g[rows], w[rows]).max())
            other = np.ones(len(g), bool)
            other[rows] = False
            assert np.array_equal(g[other], w[other]), k
        else:
            assert np.array_equal(g, w), k


def run_refine(pipe, cfg, step):
    r = MCMCRefiner(cfg)
    out = r.finish_step(step, pipe, 1e-4)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("n,dead_frac", [(3000, 0.2), (50_000, 0.5), (61, None)])
def test_relocation_against_the_restatement(n, dead_frac):
    rng = np.random.default_rng(n)
    logits = rng.uniform(-3, 3, n)
    if dead_frac is None:                      # one live Gaussian drawn 60 times: the ratio clamps at 51
        logits[:] = -9.0
        logits[17] = 1.5
    else:
        logits[rng.uniform(size=n) < dead_frac] = -8.0
    pipe = make_pipe(n, seed=n, logits=logits)
    p0, m0, v0 = host_state(pipe)
    o = dev_sigmoid(p0["opacities"])
    cfg = MCMCConfig(refine_start=0, refine_every=1, cap_max=n, noise_lr=0.0, seed=n)   # relocation only
    new_p, new_m, new_v, info = run_refine(pipe, cfg, 700)
    assert new_p is pipe.p and info["added"] == 0 and info["n"] == n
    got_s = info["relocation_samples"].cpu().numpy()
    want = ref.relocate(p0, m0, v0, o, 700, n, 0.005, samples=got_s)
    assert info["relocated"] == want["n_dead"] == len(want["dead"]) > 0
    check_samples(got_s, want["cdf"], want["cdf"], want["u"])   # the device's cdf is checked in the plan test
    if dead_frac is None:
        assert (got_s == 17).all() and want["counts"][17] == 60
    rows = np.nonzero(want["counts"])[0]
    gp, gm, gv = to_np(new_p), to_np(new_m), to_np(new_v)
    check_update(gp, p0, rows)
    for k in NAMES:                            # copied rows: bit-exact copies of the device's updated rows
        assert np.array_equal(gp[k][want["dead"]], gp[k][got_s]), k
        assert np.array_equal(gm[k], m0[k]) and np.array_equal(gv[k], v0[k]), k   # zeroed and untouched


@pytest.mark.parametrize("n", [2000, 40_000])
def test_growth_against_the_restatement(n):
    rng = np.random.default_rng(n + 1)
    pipe = make_pipe(n, seed=n + 1, logits=rng.uniform(-2, 3, n))       # nothing dead
    p0, m0, v0 = host_state(pipe)
    o = dev_sigmoid(p0["opacities"])
    cfg = MCMCConfig(refine_start=0, refine_every=1, cap_max=10 * n, noise_lr=0.0, seed=5)
    new_p, new_m, new_v, info = run_refine(pipe, cfg, 1200)
    assert info["relocated"] == 0 and info["added"] == grow_count(n, 10 * n) and info["n"] == n + info["added"]
    got_s = info["growth_samples"].cpu().numpy()
    wp, wm, wv, winfo = ref.grow(p0, m0, v0, o, 1200, 5, 0.005, 10 * n, samples=got_s)
    check_samples(got_s, winfo["cdf"], winfo["cdf"], winfo["u"])
    rows = np.nonzero(winfo["counts"])[0]
    gp, gm, gv = to_np(new_p), to_np(new_m), to_np(new_v)
    check_update({k: t[:n] for k, t in gp.items()}, {k: t[:n] for k, t in wp.items()}, rows)
    for k in NAMES:
        assert np.array_equal(gp[k][n:], gp[k][got_s]), k               # appended: copies of the updated rows
        assert np.array_equal(gm[k], wm[k]) and np.array_equal(gv[k], wv[k]), k   # kept, and zero when appended


def test_edge_cases():
    cfg = dict(refine_start=0, refine_every=1, noise_lr=0.0)
    # n = 0
    pipe = make_pipe(0)
    out = run_refine(pipe, MCMCConfig(**cfg), 10)
    assert out[0] is pipe.p and out[3]["n"] == 0 and out[3]["relocated"] == 0
    # no dead, cap reached: nothing changes
    pipe = make_pipe(500, logits=np.full(500, 0.5))
    before = [t.clone() for t in (pipe.param_flat, pipe.adam_m, pipe.adam_v)]
    out = run_refine(pipe, MCMCConfig(cap_max=500, **cfg), 10)
    assert out[3]["relocated"] == 0 and out[3]["added"] == 0 and out[0] is pipe.p
    assert all(torch.equal(a, b) for a, b in zip(before, (pipe.param_flat, pipe.adam_m, pipe.adam_v)))
    # above the cap: neither grows nor shrinks
    out = run_refine(pipe, MCMCConfig(cap_max=100, **cfg), 10)
    assert out[3]["n"] == 500 and out[0] is pipe.p
    # all dead (T = 0 for the relocation): nothing is relocated; growth still draws from the faint opacities
    pipe = make_pipe(400, logits=np.full(400, -9.0))
    before = pipe.param_flat.clone()
    out = run_refine(pipe, MCMCConfig(cap_max=400, **cfg), 10)
    assert out[3]["relocated"] == 0 and torch.equal(before, pipe.param_flat)
    out = run_refine(pipe, MCMCConfig(cap_max=1000, **cfg), 10)
    assert out[3]["added"] == 20 and out[3]["n"] == 420
    # every opacity exactly 0: both phases do nothing
    pipe = make_pipe(400, logits=np.full(400, -200.0))
    before = pipe.param_flat.clone()
    out = run_refine(pipe, MCMCConfig(cap_max=1000, **cfg), 10)
    assert out[3]["relocated"] == 0 and out[3]["added"] == 0 and torch.equal(before, pipe.param_flat)


# ---- per-step kernels ---------------------------------------------------------------------------------------------

def test_regulariser_within_its_fp32_bound():
    n = 100_003
    pipe = make_pipe(n, seed=9)
    L = capi.lib()
    g = torch.from_numpy(np.random.default_rng(1).standard_normal(n * 4).astype(np.float32) * 1e-6).to(DEV)
    go, gs = g[:n].clone(), g[n:].reshape(n, 3).clone()
    go0, gs0 = go.cpu().numpy().astype(np.float64), gs.cpu().numpy().astype(np.float64)
    co, cs = np.float32(0.01 / n), np.float32(0.02 / (3 * n))
    capi.check(L.gsb_mcmc_regularize(n, capi.ptr(pipe.p["opacities"]), capi.ptr(pipe.p["scales"]), float(co),
                                     float(cs), capi.ptr(go), capi.ptr(gs), capi.stream()))
    o = dev_sigmoid(pipe.p["opacities"].cpu().numpy()).astype(np.float64)
    s = pipe.p["scales"].cpu().numpy()
    xo, xs = ref.regularizer_grad(o, s, 0.01, 0.02)
    xo, xs = xo * (float(co) * n / 0.01), xs * (float(cs) * 3 * n / 0.02)   # the fp32 coefficients the kernel takes
    wo, ws = go0 + xo, gs0 + xs
    # opacity: 1 - o, o (1 - o), coef * that, the sum: at most 4 roundings of the term and one of the result
    assert (np.abs(go.cpu().numpy() - wo) <= U * (np.abs(wo) + 4.1 * np.abs(xo))).all()
    # scale: expf (<= 2 ulp = 4 U), the product and the sum
    assert (np.abs(gs.cpu().numpy() - ws) <= U * (np.abs(ws) + 5.1 * np.abs(xs))).all()


def test_noise_within_its_fp32_bound():
    n, step, seed, scale = 100_003, 321, 99, 0.08
    rng = np.random.default_rng(4)
    logits = rng.uniform(-9, 2, n)
    pipe = make_pipe(n, seed=4, logits=logits)
    p0 = {k: t.cpu().numpy().astype(np.float64) for k, t in pipe.p.items()}
    capi.check(capi.lib().gsb_mcmc_add_noise(n, capi.ptr(pipe.p["opacities"]), capi.ptr(pipe.p["scales"]),
                                             capi.ptr(pipe.p["quats"]), seed & 0xffffffff, seed >> 32, step, scale,
                                             capi.ptr(pipe.p["means"]), capi.stream()))
    got = pipe.p["means"].cpu().numpy().astype(np.float64)
    o = dev_sigmoid(logits.astype(np.float32)).astype(np.float64)
    z = ref.normals(ref.draws(n, seed, step, ref.NOISE_TAG))
    delta, _ = ref.noise_delta(o, p0["scales"], p0["quats"], z, scale)
    want = p0["means"] + delta
    # First-order bound from the kernel's fp32 operations: R from q / |q| has absolute errors <= 32 U per entry;
    # exp(2 s) (2 ulp) and the products / sums of Sigma v take <= 12 U relative per term; each normal is within 2e-6
    # (test_philox_words_and_normals); the gate x = (1 - o) - 0.995f, -100 x, expf, 1 + e, the reciprocal, then
    # gate * scale and z * c: relative error <= 100 (1 - gate) U (|1 - o| + 2 |x|) + 9 U; the final add: U |result|.
    gate = ref.noise_gate(o)
    x = np.abs((1 - o) - float(np.float32(0.995)))
    c = gate * float(np.float32(scale))
    v = z * c[:, None]
    dv = 2e-6 * c[:, None] + np.abs(v) * (100 * (1 - gate) * U * (np.abs(1 - o) + 2 * x) + 9 * U)[:, None]
    R = np.abs(ref.quat_to_rotmat(p0["quats"]))
    e = np.exp(2 * p0["scales"])
    A = R + 32 * U
    hi = np.einsum("nak,nk,nbk,nb->na", A, e, A, np.abs(v) + dv) * (1 + 12 * U)
    lo = np.einsum("nak,nk,nbk,nb->na", R, e, R, np.abs(v))
    bound = (hi - lo) + U * np.abs(want) * 1.0001
    err = np.abs(got - want)
    assert (err <= bound).all(), (err / bound).max()
    assert (np.abs(delta) > 0).any()


# ---- the trainer --------------------------------------------------------------------------------------------------

def _problem(n=4000, dead=400):
    from test_gpu_trainer import _cams, make_problem
    p, c2w, gts, intr, H, W = make_problem(n=n)
    p["opacities"][:dead] = -8.0                         # faint from the start: relocated at the first refinement
    return {k: torch.from_numpy(v) for k, v in p.items()}, _cams(c2w, H, W, intr), torch.from_numpy(gts).to(DEV)


def _mcmc(**kw):
    c = dict(refine_start=4, refine_every=5, refine_stop=10 ** 6, cap_max=4600, max_steps=200, seed=11)
    c.update(kw)
    return MCMCConfig(**c)


def _train(tr, cams, gts, steps, views=1, after=None):
    losses, counts, infos = [], [], []
    for step in range(1, steps + 1):
        if views == 1:
            v = (step - 1) % len(cams)
            loss = tr.step(cams[v], gts[v], step)
            losses.append(float(loss[0]))
        else:
            vs = [((step - 1) * views + b) % len(cams) for b in range(views)]
            loss = tr.step([cams[v] for v in vs], gts[vs], step)
            losses.append(float(loss[:, 0].mean()))
        if after is not None:
            after(tr, step)
        counts.append(tr.n)
        infos.append(tr.last_info)
    return np.array(losses), np.array(counts), infos


def test_trainer_equals_plain_trainer_with_finish_step():
    from test_gpu_trainer import refine_config
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts = _problem()
    cfg = _mcmc(noise_lr=0.0, opacity_reg=0.0, scale_reg=0.0)
    a = SplatTrainer(params, cfg, device=DEV, sh_degree_interval=5)
    la, ca, _ = _train(a, cams, gts, 22)
    plain = SplatTrainer(params, refine_config(warmup_length=10 ** 6, max_steps=cfg.max_steps), device=DEV,
                         sh_degree_interval=5)
    refiner = MCMCRefiner(cfg)

    def after(tr, step):
        tr._adopt(*refiner.finish_step(step, tr.pipe, tr.lr["means"]))
        d = tr.densifier                      # the plain trainer's statistics are sized by the old count
        d.xys_grad_norm = d.vis_counts = d.max_2d_size = None
    lb, cb, _ = _train(plain, cams, gts, 22, after=after)
    assert np.array_equal(ca, cb) and ca[-1] > ca[0]
    # the loss value is a float atomic sum over tiles (ssim.cu): its last bits vary from run to run; the gradient,
    # and with it every parameter, does not depend on it
    assert np.abs(la - lb).max() <= 1e-6
    for x, y in ((a.pipe.param_flat, plain.pipe.param_flat), (a.pipe.adam_m, plain.pipe.adam_m),
                 (a.pipe.adam_v, plain.pipe.adam_v)):
        assert torch.equal(x, y)


def test_regulariser_is_exactly_its_gradient_in_the_step():
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts = _problem()
    on = SplatTrainer(params, _mcmc(noise_lr=0.0, opacity_reg=0.3, scale_reg=0.2), device=DEV)
    off = SplatTrainer(params, _mcmc(noise_lr=0.0, opacity_reg=0.0, scale_reg=0.0), device=DEV)
    p0 = {k: on.pipe.p[k].clone() for k in ("opacities", "scales")}
    on.step(cams[0], gts[0], 1)
    off.step(cams[0], gts[0], 1)
    pp, n = off.pipe, off.n
    want = off.pipe.grad_flat.clone()
    g = flat_views(want, pp.offs)
    capi.check(capi.lib().gsb_mcmc_regularize(n, capi.ptr(p0["opacities"]), capi.ptr(p0["scales"]), 0.3 / n,
                                              0.2 / (3 * n), capi.ptr(g["opacities"]), capi.ptr(g["scales"]),
                                              capi.stream()))
    assert torch.equal(on.pipe.grad_flat, want)
    diff = flat_views(on.pipe.grad_flat != off.pipe.grad_flat, pp.offs)
    assert bool(diff["opacities"].any()) and bool(diff["scales"].any())
    assert not any(bool(diff[k].any()) for k in ("means", "quats", "coeffs"))


def test_seeded_runs_are_bit_identical():
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts = _problem()
    runs = []
    for seed in (11, 11, 12):
        tr = SplatTrainer(params, _mcmc(seed=seed), device=DEV)
        losses, counts, _ = _train(tr, cams, gts, 21)
        runs.append((losses, counts, tr.pipe.param_flat.clone(), tr.pipe.adam_m.clone()))
    assert np.abs(runs[0][0] - runs[1][0]).max() <= 1e-6 and np.array_equal(runs[0][1], runs[1][1])
    assert torch.equal(runs[0][2], runs[1][2]) and torch.equal(runs[0][3], runs[1][3])
    assert not torch.equal(runs[0][2], runs[2][2])          # another seed draws other numbers


def test_long_run_follows_the_count_trajectory_under_the_cap():
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts = _problem()
    cfg = _mcmc(refine_start=100, refine_every=100, refine_stop=1400, cap_max=5500, max_steps=1500)
    tr = SplatTrainer(params, cfg, device=DEV)
    losses, counts, infos = _train(tr, cams, gts, 1500)
    n, relocated = 4000, 0
    for step in range(1, 1501):
        if 100 < step < 1400 and step % 100 == 0:
            n += grow_count(n, 5500)
            relocated += infos[step - 1]["relocated"]
            assert infos[step - 1]["refined"]
        assert counts[step - 1] == n, step
    assert counts.max() == 5500 and relocated >= 400
    assert all(bool(torch.isfinite(t).all()) for t in (tr.pipe.param_flat, tr.pipe.adam_m, tr.pipe.adam_v))
    assert np.isfinite(losses).all() and losses[-100:].mean() < losses[:20].mean()


@pytest.mark.parametrize("views,antialiased", [(2, False), (1, True), (2, True)])
def test_views_and_antialiased(views, antialiased):
    from opensplat_b200.trainer import SplatTrainer
    params, cams, gts = _problem()
    tr = SplatTrainer(params, _mcmc(), device=DEV, views_per_step=views, antialiased=antialiased)
    losses, counts, infos = _train(tr, cams, gts, 21, views=views)
    assert counts[-1] == 4600 and infos[4]["relocated"] >= 400        # refinements at 5, 10, 15 (capped), 20
    assert np.isfinite(losses).all() and bool(torch.isfinite(tr.pipe.param_flat).all())
    again = SplatTrainer(params, _mcmc(), device=DEV, views_per_step=views, antialiased=antialiased)
    _train(again, cams, gts, 21, views=views)
    assert torch.equal(again.pipe.param_flat, tr.pipe.param_flat)


def _run_parallel(nproc, port):
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(nproc),
                        "--master-addr", "127.0.0.1", "--master-port", str(port),
                        os.path.join(ROOT, "tools", "check_parallel_trainer.py"), "--mcmc"],
                       capture_output=True, text=True, timeout=900)
    print(r.stdout[-4000:])
    if r.returncode != 0:
        print(r.stderr[-6000:])
    assert r.returncode == 0 and "check_ok=True" in r.stdout
    return r.stdout


def test_parallel_mcmc_world1_equals_the_plain_run():
    out = _run_parallel(1, 29561)
    assert "plain_trainer_bit_identical=True" in out


def test_parallel_mcmc_2gpu_replicas_in_sync():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = _run_parallel(2, 29563)
    assert "replicas_in_sync=True" in out
