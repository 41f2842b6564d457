"""A float64 restatement of the 3DGS-MCMC strategy (DESIGN.md D20) over numpy arrays: Philox4x32-10, the uniforms and
normals, sampling by the inclusive weight scan, the relocation update, relocation and growth of a parameter set with
its Adam moments, the regulariser gradient and the position noise.  Opacities `o` are taken as given fp32 values (the
device's 1.f / (1.f + expf(-logit))), so a test can hand in the bits the kernels see."""
import math

import numpy as np

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF
RATIO_MAX = 51
RELOCATE_TAG, GROW_TAG, NOISE_TAG = 1, 2, 0


def philox(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 over arrays (broadcast): returns the four output words as uint64 arrays < 2^32."""
    c = [np.asarray(x, dtype=np.uint64) & MASK for x in (c0, c1, c2, c3)]
    c = list(np.broadcast_arrays(*c))
    k0, k1 = np.uint64(k0 & MASK), np.uint64(k1 & MASK)
    for r in range(10):
        if r:
            k0, k1 = np.uint64((int(k0) + W0) & MASK), np.uint64((int(k1) + W1) & MASK)
        p0 = np.uint64(M0) * c[0]
        p1 = np.uint64(M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & np.uint64(MASK), (p0 >> np.uint64(32)) ^ c[3] ^ k1,
             p0 & np.uint64(MASK)]
    return c


def seed_key(seed):
    return seed & MASK, seed >> 32


def draws(count, seed, step, tag):
    """The words of counters (j, step, tag, 0), j < count, as a [count,4] uint64 array."""
    k0, k1 = seed_key(seed)
    return np.stack(philox(np.arange(count), step, tag, 0, k0, k1), -1)


def uniform(x0, x1):
    return ((x0 >> np.uint64(5)).astype(np.float64) * 2.0 ** 26 + (x1 >> np.uint64(6)).astype(np.float64)) * 2.0 ** -53


def box_muller(a, b):
    """(z_cos, z_sin) of the exact fp32 uniforms u1 = ((a >> 8) + 1) 2^-24, u2 = (b >> 8) 2^-24, in fp64."""
    u1 = ((a >> np.uint64(8)) + np.uint64(1)).astype(np.float64) * 2.0 ** -24
    u2 = (b >> np.uint64(8)).astype(np.float64) * 2.0 ** -24
    rad = np.sqrt(-2.0 * np.log(u1))
    return rad * np.cos(2 * np.pi * u2), rad * np.sin(2 * np.pi * u2)


def normals(words):
    """The three normals [count,3] of [count,4] words: z0, z1 from (x0, x1), z2 from (x2, x3)."""
    z0, z1 = box_muller(words[:, 0], words[:, 1])
    z2, _ = box_muller(words[:, 2], words[:, 3])
    return np.stack([z0, z1, z2], -1)


# ---- sampling -----------------------------------------------------------------------------------------------------

def weights(o, min_opacity=None):
    """w_i = o_i in fp64; with min_opacity (relocation) the dead ones (o <= min_opacity) weigh 0."""
    w = np.asarray(o, dtype=np.float32).astype(np.float64)
    if min_opacity is not None:
        w = np.where(np.asarray(o, np.float32) <= np.float32(min_opacity), 0.0, w)
    return w


def scan_bound(cdf):
    """A certified bound on |c_i - c_i'| between two fp64 left-to-right-grouped inclusive scans of the same
    non-negative weights: each partial sum takes at most n roundings of relative size 2^-53 on values <= T, so each is
    within n 2^-53 T (1 + n 2^-53) of the exact sum; twice that bounds the difference of two such scans."""
    n = len(cdf)
    if n == 0:
        return 0.0
    g = n * 2.0 ** -53
    return 2.0 * g * (1.0 + g) * float(cdf[-1])


def sample(cdf, u):
    """The smallest i with cdf[i] > u T, T = cdf[-1]."""
    return np.searchsorted(cdf, u * cdf[-1], side="right")


def draw_samples(cdf, m, seed, step, tag):
    """(samples, u): m draws of counters (j, step, tag, 0) from the scan cdf."""
    w = draws(m, seed, step, tag)
    u = uniform(w[:, 0], w[:, 1])
    return sample(cdf, u), u


# ---- the relocation update ----------------------------------------------------------------------------------------

def binom(n, k):
    return float(math.comb(n, k))


def relocation_D(alpha, r):
    """D = sum_{k=0}^{r-1} (-1)^k C(r, k+1) alpha^(k+1) / sqrt(k+1), in the kernel's order (fp64)."""
    D = np.zeros_like(alpha)
    ap = alpha.copy()
    b = float(r)
    for k in range(r):
        t = b * ap / math.sqrt(k + 1)
        D = D - t if k & 1 else D + t
        ap = ap * alpha
        b = b * float(r - k - 1) / float(k + 2)
    return D


def ratio_update(o, s, r, min_opacity):
    """The new (logit, log-scales) of rows with opacity o (fp32), log-scales s [m,3] (fp32), ratio r [m] (ints >= 1):
    fp64, rounded once to fp32.  Returns (logit [m] f32, scales [m,3] f32)."""
    o = np.asarray(o, np.float32).astype(np.float64)
    s = np.asarray(s, np.float32).astype(np.float64)
    r = np.asarray(r)
    logit = np.empty(len(o), np.float32)
    scales = np.empty(s.shape, np.float32)
    for rv in np.unique(r):
        m = r == rv
        with np.errstate(divide="ignore"):       # o = 1: log1p(-1) = -inf, alpha = 1
            alpha = -np.expm1(np.log1p(-o[m]) / float(rv))
        D = relocation_D(alpha, int(rv))
        a = np.minimum(np.maximum(alpha, float(np.float32(min_opacity))), 1.0 - 2.0 ** -23)
        logit[m] = (np.log(a) - np.log1p(-a)).astype(np.float32)
        scales[m] = (s[m] + np.log(o[m] / D)[:, None]).astype(np.float32)
    return logit, scales


def ratio_of(counts):
    return np.minimum(counts + 1, RATIO_MAX)


# ---- relocation and growth of a set ------------------------------------------------------------------------------

def relocate(params, adam_m, adam_v, o, step, seed, min_opacity, samples=None):
    """In place on dicts of [n,...] arrays (opacities [n,1] logits, scales [n,3]); o: the fp32 opacities.  Returns
    {n_dead, samples, dead, cdf, u} (samples None when nothing was relocated).  `samples` given: those indices
    instead of the drawn ones (a test hands in the device's draws, checked separately)."""
    n = len(o)
    cdf = np.cumsum(weights(o, min_opacity))
    dead = np.nonzero(np.asarray(o, np.float32) <= np.float32(min_opacity))[0]
    out = {"n_dead": len(dead), "dead": dead, "cdf": cdf, "samples": None, "u": None}
    if n == 0 or len(dead) == 0 or cdf[-1] == 0:
        return out
    drawn, u = draw_samples(cdf, len(dead), seed, step, RELOCATE_TAG)
    samples = drawn if samples is None else np.asarray(samples)
    counts = np.bincount(samples, minlength=n)
    rows = np.nonzero(counts)[0]
    lg, sc = ratio_update(np.asarray(o)[rows], params["scales"][rows], ratio_of(counts[rows]), min_opacity)
    params["opacities"][rows, 0] = lg
    params["scales"][rows] = sc
    for mom in (adam_m, adam_v):
        for t in mom.values():
            t[rows] = 0
    for t in params.values():
        t[dead] = t[samples]
    out.update(samples=samples, u=u, counts=counts)
    return out


def grow_count(n, cap_max):
    return max(0, min(cap_max, int(1.05 * n)) - n)


def grow(params, adam_m, adam_v, o, step, seed, min_opacity, cap_max, samples=None):
    """Returns (params, adam_m, adam_v, info): new dicts with the appended rows (the sampled rows updated in place
    first; appended moments zero, the sampled rows' moments kept).  o: the fp32 opacities after relocation;
    `samples` as in relocate()."""
    n = len(o)
    n_new = grow_count(n, cap_max)
    cdf = np.cumsum(weights(o))
    info = {"added": 0, "cdf": cdf, "samples": None, "u": None}
    if n_new == 0 or n == 0 or cdf[-1] == 0:
        return params, adam_m, adam_v, info
    drawn, u = draw_samples(cdf, n_new, seed, step, GROW_TAG)
    samples = drawn if samples is None else np.asarray(samples)
    counts = np.bincount(samples, minlength=n)
    rows = np.nonzero(counts)[0]
    lg, sc = ratio_update(np.asarray(o)[rows], params["scales"][rows], ratio_of(counts[rows]), min_opacity)
    params["opacities"][rows, 0] = lg
    params["scales"][rows] = sc
    new_p = {k: np.concatenate([t, t[samples]]) for k, t in params.items()}
    new_m = {k: np.concatenate([t, np.zeros_like(t[samples])]) for k, t in adam_m.items()}
    new_v = {k: np.concatenate([t, np.zeros_like(t[samples])]) for k, t in adam_v.items()}
    info.update(added=n_new, samples=samples, u=u, counts=counts)
    return new_p, new_m, new_v, info


def refines(step, refine_start=500, refine_stop=25_000, refine_every=100):
    return refine_start < step < refine_stop and step % refine_every == 0


# ---- per step ----------------------------------------------------------------------------------------------------

def regularizer_grad(o, s, opacity_reg, scale_reg):
    """The gradients of opacity_reg mean|o| + scale_reg mean|exp s| w.r.t. the logits [n] and log-scales [n,3]."""
    o = np.asarray(o, np.float64)
    n = len(o)
    return opacity_reg * o * (1 - o) / n, scale_reg * np.exp(np.asarray(s, np.float64)) / (3 * n)


def quat_to_rotmat(q):
    q = np.asarray(q, np.float64)
    q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def noise_gate(o):
    """sigma_100((1 - o) - 0.995f) of fp32 opacities, with the fp32 constant the kernel uses."""
    o = np.asarray(o, np.float32).astype(np.float64)
    return 1.0 / (1.0 + np.exp(-100.0 * ((1.0 - o) - float(np.float32(0.995)))))


def noise_delta(o, s, quats, z, noise_scale):
    """Sigma (z sigma_100(1 - o - 0.995) noise_scale), Sigma = R diag(exp(2 s)) R^T; returns (delta [n,3], and the
    magnitudes sum_b |Sigma|_ab |v_b| with |Sigma|_ab = sum_k |R_ak R_bk| exp(2 s_k), for error bounds)."""
    R = quat_to_rotmat(quats)
    e = np.exp(2.0 * np.asarray(s, np.float64))
    v = z * (noise_gate(o) * float(np.float32(noise_scale)))[:, None]
    sig = np.einsum("nak,nk,nbk->nab", R, e, R)
    mag = np.einsum("nak,nk,nbk->nab", np.abs(R), e, np.abs(R))
    return np.einsum("nab,nb->na", sig, v), np.einsum("nab,nb->na", mag, np.abs(v))
