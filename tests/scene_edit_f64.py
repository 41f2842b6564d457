"""Float64 restatement of the topology-edit kernels of csrc/densify.cu (classify, compaction, means_scales) and the
scene packers of csrc/export.cu (PLY pack / unpack, .splat order keys and rows), with a per-element error bound that
follows each kernel's fp32 operation tree and a certificate for every threshold decision.

Bounds.  A value V carries its float64 value v (of the exact operation on the fp32 inputs the kernel reads) and a
first-order bound b on |fp32 evaluation - v|.  Each IEEE operation (+, -, *, /, sqrt) adds u |result| + ETA (u =
2^-24, ETA = 2^-150 for a subnormal result), except when its operands are exact (b = 0) and the exact result is an
fp32 number: then IEEE rounding returns it and the result stays exact.  expf adds 2 ulp (<= 4 u |result|) and logf
1 ulp (<= 2 u |result|), the CUDA Programming Guide's bounds for builds without fast math; expf(0) = 1 and logf(1) = 0
exactly (the guide's special values).  A rounding taken on its own dominates the same operation fused into an FMA,
so the bound holds whether nvcc contracts mul+add pairs or not (densify.cu is built with contraction, export.cu
without).  Tests compare with C = 2 times the bound, which covers the second-order terms.

Decisions.  classify_one compares mx = max expf(s), avg = ((gn / vc) 0.5) max_dim, sigmoid(o) = 1 / (1 + expf(-o))
and the split child's max expf(logf(expf(s) / size_fac)) against the fp32 thresholds the C ABI receives.  A
comparison is certified when the distance to its threshold exceeds C b, or when the value is not finite (vc = 0 gives
gn / 0 = NaN or inf, exact).  max2DSize is an exact input, so its two comparisons are always certified.  A parent is
certified when every comparison its outcome can depend on is.

Compaction.  src_map = cat(originals, split sample 0, split sample 1, dups)[~culls] with the kind in bits 30-31,
split_rank = rank among split parents, counts = n_splits, kept originals, kept split parents, kept dups, new_n,
n_dups, 0, 0 -- plain numpy, exact.

Export (export.cu is built --fmad=false, so every fp32 operation is rounded on its own).  The PLY rows and the
keepCrs means are reproduced bit for bit by numpy fp32 arithmetic (IEEE, as the device's); the keepCrs scales
log(exp(s) / scale) and log(scale exp(s)) go through expf / logf and get a bound.  The .splat key is
((e0 + e1) + e2) / (1 + expf(-o)), e = expf(s) (/ scale with keepCrs).  A .splat byte is trunc(x) of x =
clamp(dc C0 + 0.5, 0, 1) 255, clamp(255 / (1 + expf(-o)), 0, 255) or clamp(q 128 + 128, 0, 255); it is certified
when x lies further than C b from every integer (or is exact), otherwise both neighbouring bytes are accepted."""
import numpy as np

U = 2.0 ** -24
ETA = 2.0 ** -150
EXP_ULP = 4.0            # expf: 2 ulp <= 4 u |result|
LOG_ULP = 2.0            # logf: 1 ulp <= 2 u |result|
C = 2.0
KIND_SHIFT = 30
SH_C0 = float(np.float32(0.28209479177387814))


def f32(x):
    return np.asarray(x, np.float32).astype(np.float64)


class V:
    """Float64 value v with a first-order bound b on the error of its fp32 evaluation."""
    __slots__ = ("v", "b")

    def __init__(self, v, b=None):
        self.v = np.asarray(v, np.float64)
        self.b = np.zeros_like(self.v) if b is None else np.asarray(b, np.float64)

    @staticmethod
    def of(x):
        return x if isinstance(x, V) else V(f32(x))

    def _round(self, v, b, exact_in):
        with np.errstate(over="ignore", invalid="ignore"):
            fits = np.isfinite(v) & (v.astype(np.float32).astype(np.float64) == v)
        return V(v, np.where(exact_in & fits, 0.0, b + U * np.abs(v) + ETA))

    def __add__(self, o):
        o = V.of(o)
        return self._round(self.v + o.v, self.b + o.b, (self.b == 0) & (o.b == 0))

    __radd__ = __add__

    def __sub__(self, o):
        o = V.of(o)
        return self._round(self.v - o.v, self.b + o.b, (self.b == 0) & (o.b == 0))

    def __rsub__(self, o):
        return V.of(o) - self

    def __mul__(self, o):
        o = V.of(o)
        with np.errstate(invalid="ignore"):     # inf (x / 0) times a zero bound
            b = np.abs(self.v) * o.b + np.abs(o.v) * self.b
        return self._round(self.v * o.v, b, (self.b == 0) & (o.b == 0))

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = V.of(o)
        with np.errstate(divide="ignore", invalid="ignore"):
            v = self.v / o.v
            b = (self.b + np.abs(v) * o.b) / np.abs(o.v)
        return self._round(v, b, (self.b == 0) & (o.b == 0))

    def __rtruediv__(self, o):
        return V.of(o) / self

    def __neg__(self):
        return V(-self.v, self.b)

    def __getitem__(self, i):
        return V(self.v[i], self.b[i])


def sqrt_(a):
    v = np.sqrt(a.v)
    with np.errstate(divide="ignore", invalid="ignore"):
        lin = np.where(v > 0, a.b / (2 * np.maximum(v, 1e-300)), np.inf)
    return a._round(v, np.minimum(lin, np.sqrt(a.b)), a.b == 0)


def exp_(a):
    with np.errstate(over="ignore"):
        v = np.exp(a.v)
    exact = (a.b == 0) & (a.v == 0)
    return V(v, np.where(exact, 0.0, v * a.b + EXP_ULP * U * v + ETA))


def log_(a):
    with np.errstate(divide="ignore"):
        v = np.log(a.v)
    exact = (a.b == 0) & (a.v == 1)
    return V(v, np.where(exact, 0.0, a.b / a.v + LOG_ULP * U * np.abs(v) + ETA))


def vmax(*xs):
    """fmaxf of fp32 evaluations: at least the arg-max's value minus its bound, at most max (v_k + b_k)."""
    v = np.maximum.reduce([x.v for x in xs])
    b_arg = np.maximum.reduce([np.where(x.v == v, x.b, 0.0) for x in xs])
    over = np.maximum.reduce([x.v + C * x.b for x in xs]) - v     # so that C b covers the largest v_k + C b_k
    return V(v, np.maximum(b_arg, over / C))


def vclamp(x, lo, hi):
    """fminf(fmaxf(x, lo), hi): exact at a bound the value certainly passes, else 1-Lipschitz."""
    v = np.clip(x.v, lo, hi)
    b = np.where((x.v - C * x.b >= hi) | (x.v + C * x.b <= lo), 0.0, x.b)
    return V(v, b)


def certified(x, thresh):
    """The comparison of x with a threshold decides the same way for every value within C b (or x is exact)."""
    with np.errstate(invalid="ignore"):
        return ~np.isfinite(x.v) | (x.b == 0) | (np.abs(x.v - thresh) > C * x.b)


# ---- classify ---------------------------------------------------------------------------------------------------
THRESHOLDS = ("densify_grad_thresh", "densify_size_thresh", "split_screen_size", "cull_alpha_thresh",
              "cull_scale_thresh", "cull_screen_size", "size_fac")


def cfg32(cfg):
    """The fp32 thresholds gsb_densify_classify receives (float arguments of the C ABI)."""
    return {k: float(np.float32(getattr(cfg, k))) for k in THRESHOLDS}


def quantities(scales, opacities, gn, vc, max_dim, size_fac):
    """mx, avg, sigmoid(o) and the split child's max scale of each parent, as V."""
    s = V(f32(scales).reshape(-1, 3))
    e = [exp_(s[:, k]) for k in range(3)]
    mx = vmax(*e)
    avg = ((V(f32(gn).reshape(-1)) / V(f32(vc).reshape(-1))) * 0.5) * float(np.float32(max_dim))
    sig = 1.0 / (1.0 + exp_(-V(f32(opacities).reshape(-1))))
    fac = float(np.float32(size_fac))
    mxc = vmax(*[exp_(log_(ek / fac)) for ek in e])
    return {"mx": mx, "avg": avg, "sig": sig, "mxc": mxc}


def classify(scales, opacities, gn, vc, m2d, max_dim, cfg, check_split_screen, check_huge, check_cull_screen):
    """classify_one in float64.  m2d None = the ABI's max_2d_size NULL (read as 0).  Returns a dict of the decision
    vectors split, dup, keep_self, keep_split, keep_dup, the certificate `cert`, and the quantities."""
    t = cfg32(cfg)
    q = quantities(scales, opacities, gn, vc, max_dim, t["size_fac"])
    mx, avg, sig, mxc = q["mx"], q["avg"], q["sig"], q["mxc"]
    n = mx.v.shape[0]
    m2 = np.zeros(n) if m2d is None else f32(m2d).reshape(-1)
    with np.errstate(invalid="ignore"):
        high = avg.v > t["densify_grad_thresh"]
    big = mx.v > t["densify_size_thresh"]
    screen = bool(check_split_screen) & (m2 > t["split_screen_size"])
    split = (big | screen) & high
    dup = ~big & high
    lowa = sig.v < t["cull_alpha_thresh"]
    cull_screen = bool(check_cull_screen) & (m2 > t["cull_screen_size"])
    child_screen = bool(check_cull_screen) and 0.0 > t["cull_screen_size"]
    huge_self = bool(check_huge) & ((mx.v > t["cull_scale_thresh"]) | cull_screen)
    huge_split_child = bool(check_huge) & ((mxc.v > t["cull_scale_thresh"]) | child_screen)
    huge_dup_child = bool(check_huge) & ((mx.v > t["cull_scale_thresh"]) | child_screen)
    d = {"split": split, "dup": dup, "keep_split": split & ~lowa & ~huge_split_child,
         "keep_dup": dup & ~lowa & ~huge_dup_child, "keep_self": ~lowa & ~split & ~huge_self}
    c_high, c_size = certified(avg, t["densify_grad_thresh"]), certified(mx, t["densify_size_thresh"])
    c_alpha, c_cull = certified(sig, t["cull_alpha_thresh"]), certified(mx, t["cull_scale_thresh"])
    c_child = certified(mxc, t["cull_scale_thresh"])
    maybe_high = high | ~c_high
    maybe_split = maybe_high & (big | ~c_size | screen)
    unc = ~c_high | (maybe_high & ~c_size) | ~c_alpha
    if check_huge:
        unc |= ~c_cull | (maybe_split & ~c_child)
    d["cert"] = ~unc
    d.update(q)
    return d


def compact(split, dup, keep_self, keep_split, keep_dup, **_):
    """The exact outputs of the classify kernels for given decisions: (src_map [new_n] i32, split_rank [n] i32,
    counts [8] i32)."""
    split, keep_self, keep_split, keep_dup = (np.asarray(x, bool) for x in (split, keep_self, keep_split, keep_dup))
    idx = np.arange(len(split), dtype=np.int64)
    ks = idx[keep_split]
    src = np.concatenate([idx[keep_self], ks | (1 << KIND_SHIFT), ks | (2 << KIND_SHIFT),
                          idx[keep_dup] | (3 << KIND_SHIFT)]).astype(np.uint32).view(np.int32)
    split_rank = np.where(split, np.cumsum(split) - 1, -1).astype(np.int32)
    counts = np.array([split.sum(), keep_self.sum(), keep_split.sum(), keep_dup.sum(), len(src),
                       np.asarray(dup, bool).sum(), 0, 0], np.int32)
    return src, split_rank, counts


def decisions_of(src_map, split_rank, n):
    """The decisions a kernel took, read back from its outputs (split_rank >= 0 and the kinds present in src_map).
    `dup` is only visible where the duplicate survives."""
    e = np.asarray(src_map).view(np.uint32)
    parent, kind = (e & ((1 << KIND_SHIFT) - 1)).astype(np.int64), e >> KIND_SHIFT
    out = {"split": np.asarray(split_rank)[:n] >= 0}
    for name, k in (("keep_self", 0), ("keep_split", 1), ("keep_dup", 3)):
        m = np.zeros(n, bool)
        m[parent[kind == k]] = True
        out[name] = m
    out["dup"] = out["keep_dup"].copy()
    return out


# ---- means_scales ------------------------------------------------------------------------------------------------
def means_scales(src_map, split_rank, n_splits, samples, means, scales, quats, size_fac):
    """densify_means_scales_kernel in float64: (new_means V [new_n,3], new_scales V [new_n,3]).  Survivors and
    duplicates are exact copies; child j of kind 1/2 takes sample row (kind - 1) n_splits + split_rank[parent]."""
    e = np.asarray(src_map).view(np.uint32)
    p, kind = (e & ((1 << KIND_SHIFT) - 1)).astype(np.int64), (e >> KIND_SHIFT).astype(np.int64)
    means, scales, quats = f32(means).reshape(-1, 3), f32(scales).reshape(-1, 3), f32(quats).reshape(-1, 4)
    nm_v, nm_b = means[p].copy(), np.zeros((len(p), 3))
    ns_v, ns_b = scales[p].copy(), np.zeros((len(p), 3))
    ch = np.nonzero((kind == 1) | (kind == 2))[0]
    if len(ch):
        pc = p[ch]
        row = (kind[ch] - 1) * n_splits + np.asarray(split_rank, np.int64)[pc]
        smp = f32(samples).reshape(-1, 3)[row]
        ex = [exp_(V(scales[pc, k])) for k in range(3)]
        v = [ex[k] * V(smp[:, k]) for k in range(3)]
        w, x, y, z = (V(quats[pc, k]) for k in range(4))
        for _ in range(2):   # q / |q| (model.cpp:361), then F.normalize inside quatToRotMat (max(|q|, 1e-12))
            nrm = sqrt_(((w * w + x * x) + y * y) + z * z)
            nrm = V(np.maximum(nrm.v, float(np.float32(1e-12))), nrm.b)
            w, x, y, z = w / nrm, x / nrm, y / nrm, z / nrm
        r = [[1.0 - 2.0 * (y * y + z * z), 2.0 * (x * y - w * z), 2.0 * (x * z + w * y)],
             [2.0 * (x * y + w * z), 1.0 - 2.0 * (x * x + z * z), 2.0 * (y * z - w * x)],
             [2.0 * (x * z - w * y), 2.0 * (y * z + w * x), 1.0 - 2.0 * (x * x + y * y)]]
        fac = float(np.float32(size_fac))
        for a in range(3):
            m = V(means[pc, a]) + ((r[a][0] * v[0] + r[a][1] * v[1]) + r[a][2] * v[2])
            nm_v[ch, a], nm_b[ch, a] = m.v, m.b
            s = log_(ex[a] / fac)
            ns_v[ch, a], ns_b[ch, a] = s.v, s.b
    return V(nm_v, nm_b), V(ns_v, ns_b)


# ---- export ------------------------------------------------------------------------------------------------------
def crs_means(means, scale, translation):
    """m / scale + t in fp32 (IEEE division, then addition)."""
    m = np.asarray(means, np.float32).reshape(-1, 3)
    return m / np.float32(scale) + np.asarray(translation, np.float32)


def ply_rows(means, dc, rest, opacities, scales, quats, keep_crs=False, scale=1.0, translation=(0.0, 0.0, 0.0)):
    """The PLY vertex rows [n, 14 + 3K] fp32 of fp32 numpy inputs (dc [n,3], rest [n,K-1,3]) and the keepCrs scale
    columns as V (None without keepCrs); those three columns of the fp32 rows hold the float64 value rounded."""
    n = means.shape[0]
    rest = np.asarray(rest, np.float32).reshape(n, -1, 3)
    cols = [crs_means(means, scale, translation) if keep_crs else np.asarray(means, np.float32),
            np.zeros((n, 3), np.float32), np.asarray(dc, np.float32).reshape(n, 3),
            rest.transpose(0, 2, 1).reshape(n, -1), np.asarray(opacities, np.float32).reshape(n, 1),
            np.asarray(scales, np.float32), np.asarray(quats, np.float32)]
    sc = None
    if keep_crs:
        sc = log_(exp_(V(f32(scales))) / float(np.float32(scale)))
        cols[5] = sc.v.astype(np.float32)
    return np.concatenate(cols, 1), sc


def unpack_crs(rows_means, rows_scales, scale, translation):
    """The keepCrs loader: means (m - t) scale bit for bit in fp32, scales log(scale exp(s)) as V."""
    m = (np.asarray(rows_means, np.float32) - np.asarray(translation, np.float32)) * np.float32(scale)
    return m, log_(float(np.float32(scale)) * exp_(V(f32(rows_scales))))


def splat_scales(scales, keep_crs=False, scale=1.0):
    e = [exp_(V(f32(scales).reshape(-1, 3)[:, k])) for k in range(3)]
    if keep_crs:
        e = [x / float(np.float32(scale)) for x in e]
    return e


def splat_key(scales, opacities, keep_crs=False, scale=1.0):
    """The .splat order key ((e0 + e1) + e2) / (1 + expf(-o)) as V."""
    e = splat_scales(scales, keep_crs, scale)
    return ((e[0] + e[1]) + e[2]) / (1.0 + exp_(-V(f32(opacities).reshape(-1))))


def decode_keys(keys):
    """Float keys of splat_keys_kernel's int64 encoding (ascending integer = descending float)."""
    b = ~np.asarray(keys).astype(np.uint32)
    f = np.where(b & np.uint32(0x80000000), b ^ np.uint32(0x80000000), ~b)
    return f.astype(np.uint32).view(np.float32)


def splat_bytes(dc, opacities, quats):
    """The u8 fields as V before truncation: rgb [n,3], alpha [n], quat [n,4]."""
    rgb = vclamp(V(f32(dc).reshape(-1, 3)) * SH_C0 + 0.5, 0.0, 1.0) * 255.0
    a = vclamp((1.0 / (1.0 + exp_(-V(f32(opacities).reshape(-1))))) * 255.0, 0.0, 255.0)
    q = vclamp(V(f32(quats).reshape(-1, 4)) * 128.0 + 128.0, 0.0, 255.0)
    return rgb, a, q


def splat_bytes_fp32(dc, quats):
    """rgb [n,3] and quat [n,4] bytes bit for bit: no expf on their path, every fp32 operation is IEEE."""
    f = np.float32
    rgb = np.clip(np.asarray(dc, f).reshape(-1, 3) * f(SH_C0) + f(0.5), f(0), f(1)) * f(255)
    q = np.clip(np.asarray(quats, f).reshape(-1, 4) * f(128) + f(128), f(0), f(255))
    return np.trunc(rgb).astype(np.uint8), np.trunc(q).astype(np.uint8)


def byte_check(got, x):
    """(ok [..] bool, certified [..] bool) of bytes `got` against trunc(x): a certified element must match exactly, an
    uncertified one (x within C b of an integer) may take either neighbouring byte."""
    got = np.asarray(got).astype(np.int64)
    lo, hi = np.floor(x.v - C * x.b), np.floor(x.v + C * x.b)
    cert = (lo == hi) | (x.b == 0)
    want = np.trunc(x.v).astype(np.int64)
    ok = np.where(cert, got == want, (got >= lo) & (got <= hi))
    return ok, cert


def order_check(order, key, exact_keys=None):
    """Violations of a descending order: adjacent rows whose float64 keys are certainly ascending, and, given the
    sorted fp32 keys the device compared, ties out of ascending index.  Returns (n certainly misordered, n ties out of
    index order, n uncertified adjacent pairs)."""
    order = np.asarray(order, np.int64)
    kv, kb = key.v[order], C * key.b[order]
    gap = kv[1:] - kv[:-1]
    tol = kb[1:] + kb[:-1]
    bad = int((gap > tol).sum())
    unc = int((np.abs(gap) <= tol).sum())
    ties = 0
    if exact_keys is not None:
        ks = np.asarray(exact_keys)
        tie = ks[1:] == ks[:-1]
        ties = int((tie & (order[1:] < order[:-1])).sum()) + int((ks[1:] > ks[:-1]).sum())
    return bad, ties, unc
