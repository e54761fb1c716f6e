"""Exact reference of the factor maths, and the edge corpus that drives every evaluator of it.

TEST INFRASTRUCTURE.  The factor maths -- the xyt residual and Jacobians, J_a'WJ_a / J_b'WJ_b (packed upper
triangles), J'Wr, the off-diagonal block, the robust weight w(s) and cost rho(s), the chi2 term -- exists in the host
hooks (host/graph.c) and in k_linearize / k_step, k_hessian_rebuild and k_chi2_partial.  `factor_ref` evaluates it in
mpmath at DPS digits from the double inputs taken as exact, and returns, next to every exact value, the sum of the
absolute values of its terms (the "abs" of LINEARIZE_C-style bounds: a double evaluation is within a small multiple of
u times it).  It is written on its own, without emul.py or frontcheck.linearize_ref, so that it cannot share their
mistakes.

Conventions the kernels keep:
  * r[2] = mod2pi(z[2] - (theta_b - theta_a)) in [-pi, pi); at the +-pi seam either representative is accepted
    (`factor_ref` returns both variants when the exact r[2] is within the rounding bound of the seam);
  * the off-diagonal block is J_early' W_eff J_late, "early" the pose eliminated first (smaller node2q), stored as
    [lower node id][higher node id] (transposed when the early pose has the higher id);
  * the chi2 term is 0.5 rho(s) for two-pose factors (rho = s without a loss) and s = r'Wr for priors.

`corpus()` builds the seeded edge corpus (headings at the seam, coordinates up to 1e9, ill-conditioned and 2^e-scaled
W, both losses over the whole accepted k range, both orientations and parallel factors, and the kernel shapes: a hub
of more than 64 factors, a slot of 40 or more, more than 32 dirty slots).
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field

import mpmath
import numpy as np

DPS = 60
U = 2.0 ** -53
DBL_MIN = 2.0 ** -1022
DBL_MAX = float(np.finfo(np.float64).max)
ETA = 2.0 ** -1074  # least subnormal: the absolute error of one rounding in the subnormal range
HUBER, CAUCHY = 1, 2
PACK = (0, 1, 2, 4, 5, 8)  # packed upper triangle of a row-major 3x3


# ---------------------------------------------------------------------------------------------
# exact reference
# ---------------------------------------------------------------------------------------------
def _m(x):
    return mpmath.mpf(float(x))


def loss_exact(loss, k, s):
    """(w, |w'|, rho) of the loss at s >= 0, exact (mpf inputs or doubles).  |w'| bounds the slope of w near s: at the
    Huber kink an error in s can cross k^2, so inside it is the largest slope outside, 1 / (2 k^2)."""
    k, s = mpmath.mpf(k), mpmath.mpf(s)
    k2 = k * k
    if loss == HUBER:
        if s <= k2:
            return mpmath.mpf(1), 1 / (2 * k2), s
        q = mpmath.sqrt(s)
        return k / q, k / (2 * s * q), 2 * k * q - k2
    t = s / k2
    w = 1 / (1 + t)
    return w, w * w / k2, k2 * mpmath.log1p(t)


def loss_ref(loss, k, s):
    """(w, rho) of the loss at the double s, as exact mpf values."""
    with mpmath.workdps(DPS):
        w, _, rho = loss_exact(loss, k, s)
        return w, rho


def _mm(A, B):
    return [[sum(A[i][q] * B[q][j] for q in range(3)) for j in range(3)] for i in range(3)]


def _tr(A):
    return [[A[j][i] for j in range(3)] for i in range(3)]


def _mv(A, v):
    return [sum(A[i][q] * v[q] for q in range(3)) for i in range(3)]


@dataclass
class Ref:
    """Exact values (float64 arrays rounded from DPS digits) and the sums of the absolute values of their terms."""
    val: dict = field(default_factory=dict)
    abs: dict = field(default_factory=dict)


def _put(ref, name, v, a):
    ref.val[name] = np.array([[float(x) for x in row] for row in v]) if isinstance(v[0], list) else \
        np.array([float(x) for x in v])
    ref.abs[name] = np.array([[float(x) for x in row] for row in a]) if isinstance(a[0], list) else \
        np.array([float(x) for x in a])


def factor_ref(ftype, z, W, pa, pb=None, loss=0, k=0.0, a_early=True, a_lower=True):
    """Every quantity of one factor, exact, as a list of Ref variants (two at the +-pi seam, else one).

    ftype 1 / 32 (two poses, evaluated at pa, pb; loss/k for 32) or 2 (prior at pa).  a_early: pose a is eliminated
    first (node2q[a] < node2q[b]); a_lower: a < b.  Quantities: r, Ja, Jb, s, w, rho, Weff (3x3), Da, Db (packed 6),
    ba, bb (J'Wr), H (3x3, storage convention of the kernels), chi2."""
    with mpmath.workdps(DPS):
        pi = mpmath.pi
        z = [_m(v) for v in z]
        Wm = [[_m(W[3 * i + j]) for j in range(3)] for i in range(3)]
        WA = [[abs(x) for x in row] for row in Wm]
        pa = [_m(v) for v in pa]
        two = ftype != 2
        if two:
            pb = [_m(v) for v in pb]
            ca, sa = mpmath.cos(pa[2]), mpmath.sin(pa[2])
            dx, dy = pb[0] - pa[0], pb[1] - pa[1]
            dxA, dyA = abs(pb[0]) + abs(pa[0]), abs(pb[1]) + abs(pa[1])
            v2 = z[2] - (pb[2] - pa[2])
            v2A = abs(z[2]) + abs(pb[2]) + abs(pa[2])
            r01 = [z[0] - (ca * dx + sa * dy), z[1] - (-sa * dx + ca * dy)]
            r01A = [abs(z[0]) + abs(ca) * dxA + abs(sa) * dyA, abs(z[1]) + abs(sa) * dxA + abs(ca) * dyA]
            Ja = [[-ca, -sa, -sa * dx + ca * dy], [sa, -ca, -ca * dx - sa * dy], [0, 0, -1]]
            JaA = [[abs(ca), abs(sa), abs(sa) * dxA + abs(ca) * dyA], [abs(sa), abs(ca), abs(ca) * dxA + abs(sa) * dyA],
                   [0, 0, 1]]
            Jb = [[ca, sa, 0], [-sa, ca, 0], [0, 0, 1]]
            JbA = [[abs(x) for x in row] for row in Jb]
        else:
            r01 = [z[0] - pa[0], z[1] - pa[1]]
            r01A = [abs(z[0]) + abs(pa[0]), abs(z[1]) + abs(pa[1])]
            v2 = z[2] - pa[2]
            v2A = abs(z[2]) + abs(pa[2])
        n = mpmath.floor((v2 + pi) / (2 * pi))
        r2 = v2 - 2 * pi * n
        r2A = v2A + 2 * pi * (abs(n) + 1)
        reps = [r2]
        if abs(abs(r2) - pi) <= 64 * U * r2A:  # at the seam: the other representative too
            reps.append(r2 - 2 * pi if r2 > 0 else r2 + 2 * pi)
        out = []
        for r2v in reps:
            ref = Ref()
            r = [r01[0], r01[1], r2v]
            rA = [r01A[0], r01A[1], r2A]
            X = _mv(Wm, r)
            s = sum(r[i] * X[i] for i in range(3))
            sA = sum(rA[i] * WA[i][j] * rA[j] for i in range(3) for j in range(3))
            if ftype == 32:
                w, dw, rho = loss_exact(loss, k, s)
                # s itself is formed with relative error ~u sA / s and an absolute error of a few ETA (underflow)
                wA = w + dw * (sA + 8 * ETA / U)
                rhoA = abs(rho) + w * (sA + 8 * ETA / U)
            else:
                w, wA, rho, rhoA = mpmath.mpf(1), mpmath.mpf(1), s, sA
            We = [[w * x for x in row] for row in Wm]
            WeA = [[wA * x for x in row] for row in WA]
            _put(ref, "r", r, rA)
            _put(ref, "s", [s], [sA])
            _put(ref, "w", [w], [wA])
            _put(ref, "rho", [rho], [rhoA])
            _put(ref, "Weff", We, WeA)
            if two:
                JatW, JatWA = _mm(_tr(Ja), We), _mm(_tr(JaA), WeA)
                JbtW, JbtWA = _mm(_tr(Jb), We), _mm(_tr(JbA), WeA)
                Da, DaA = _mm(JatW, Ja), _mm(JatWA, JaA)
                Db, DbA = _mm(JbtW, Jb), _mm(JbtWA, JbA)
                if a_early:
                    Hm, HA = _mm(JatW, Jb), _mm(JatWA, JbA)
                else:
                    Hm, HA = _mm(JbtW, Ja), _mm(JbtWA, JaA)
                if a_early != a_lower:  # the early pose has the higher id: stored [lower][higher]
                    Hm, HA = _tr(Hm), _tr(HA)
                _put(ref, "Ja", Ja, JaA)
                _put(ref, "Jb", Jb, JbA)
                _put(ref, "Da", [Da[i // 3][i % 3] for i in PACK], [DaA[i // 3][i % 3] for i in PACK])
                _put(ref, "Db", [Db[i // 3][i % 3] for i in PACK], [DbA[i // 3][i % 3] for i in PACK])
                _put(ref, "ba", _mv(JatW, r), _mv(JatWA, rA))
                _put(ref, "bb", _mv(JbtW, r), _mv(JbtWA, rA))
                _put(ref, "H", Hm, HA)
                _put(ref, "chi2", [rho / 2], [rhoA / 2])
            else:
                _put(ref, "Da", [Wm[i // 3][i % 3] for i in PACK], [WA[i // 3][i % 3] for i in PACK])
                _put(ref, "ba", _mv(Wm, r), _mv(WA, rA))
                _put(ref, "chi2", [s], [sA])
            out.append(ref)
        return out


# ---------------------------------------------------------------------------------------------
# checkers
# ---------------------------------------------------------------------------------------------
def excess(got: dict, refs, names=None) -> float:
    """Worst |got - exact| / (u sum|terms| + DBL_MIN) over the quantities `names` (default: all in got), for the
    variant that fits best.  A NaN anywhere gives inf."""
    best = math.inf
    for ref in refs:
        worst = 0.0
        for name in (names or got.keys()):
            g = np.asarray(got[name], dtype=np.float64)
            e = np.abs(g - ref.val[name]) / (U * ref.abs[name] + DBL_MIN)
            worst = max(worst, math.inf if np.isnan(e).any() else float(e.max(initial=0.0)))
        best = min(best, worst)
    return best


def ulps(got: float, exact) -> float:
    """Error of a double against an exact value: in ulps of the exact value where it is normal, in units of DBL_MIN
    below that (so <= 1 means an absolute error of at most DBL_MIN).  NaN gives inf."""
    if math.isnan(got):
        return math.inf
    with mpmath.workdps(DPS):
        exact = mpmath.mpf(exact)
        err = abs(mpmath.mpf(got) - exact)
        if abs(exact) < DBL_MIN:
            return float(err / DBL_MIN)
        e = int(mpmath.floor(mpmath.log(abs(exact), 2)))
        return float(err / mpmath.ldexp(1, e - 52))


# ---------------------------------------------------------------------------------------------
# the corpus
# ---------------------------------------------------------------------------------------------
def _k_list():
    kmin_normal = 2.0 ** -511  # k^2 = DBL_MIN exactly
    kmax = math.sqrt(DBL_MAX)
    while kmax * kmax <= DBL_MAX:
        kmax = math.nextafter(kmax, math.inf)
    while not (kmax * kmax <= DBL_MAX):
        kmax = math.nextafter(kmax, 0.0)
    return [5e-324, 1e-170, 1e-160, kmin_normal, 1e-3, 1.0, 1e100, 1e146, 1e154, kmax, 1e155, 1e300, DBL_MAX]


K_LIST = _k_list()
# k with k^2 subnormal whose k * k rounds above k^2: the one just above sqrt(ETA / 2) (fl(k^2) = ETA, k^2 ~ ETA / 2)
# and one in the middle of the subnormal range
K_STRADDLE = [math.nextafter(math.sqrt(ETA) * math.sqrt(0.5), 1.0), 1.6531141200240235e-162]


def loss_band(k: float, s: float) -> str:
    """Which branch of the Cauchy maths a (k, s) takes: 'normal' (k^2 and s / k^2 normal), 'k2_inf', 'k2_small'
    (zero or subnormal), 't_small' (s / k^2 zero or subnormal with s > 0), 't_inf'."""
    k2 = k * k
    if k2 > DBL_MAX:
        return "k2_inf"
    if k2 < DBL_MIN:
        return "k2_small"
    t = s / k2
    if t > DBL_MAX:
        return "t_inf"
    if s > 0 and t < DBL_MIN:
        return "t_small"
    return "normal"


def loss_rows():
    """(loss, k, r0, W00) of the isolated loss cases: r = (r0, 0, 0) exactly (two coincident poses), W = diag(W00, 1, 1),
    so the kernels form s = fl(r0 fl(W00 r0)) = `loss_s(r0, W00)`.  s = 0, exactly k^2, about one ulp either side of it,
    and 1e-30, 1, 1e20; rows where s itself would exceed DBL_MAX / 4 are left out.
    Where k^2 is below DBL_MIN, k * k can be far from k^2, so these three rows all give s = fl(k^2); there the rows with
    r0 = 1 and W00 = s put s on the doubles just below and just above the exact k^2 (`straddle`)."""
    rows = []
    up, dn = math.nextafter(1.0, 2.0), math.nextafter(1.0, 0.0)
    for loss in (HUBER, CAUCHY):
        for k in K_LIST + K_STRADDLE:
            for r0, W00 in ((0.0, 1.0), (k, 1.0), (k, up), (k, dn), (1e-15, 1.0), (1.0, 1.0), (1e10, 1.0)):
                if r0 <= math.sqrt(DBL_MAX / 4 / W00):
                    rows.append((loss, k, r0, W00))
            for s in straddle(k):
                rows.append((loss, k, 1.0, s))
    return rows


def straddle(k):
    """The positive doubles just below (or at) and just above the exact k^2, where k^2 < DBL_MIN; else none."""
    if k * k >= DBL_MIN:
        return []
    with mpmath.workdps(DPS):
        k2 = mpmath.mpf(k) ** 2
        lo = float(mpmath.floor(k2 / ETA) * ETA)
        hi = float((mpmath.floor(k2 / ETA) + 1) * ETA)
    return [v for v in (lo, hi) if v > 0]


def loss_s(r0, W00):
    return r0 * (W00 * r0)


@dataclass
class Graph:
    """A pose graph of the corpus: poses (N, 3) and factors (type, a, b, z, W (9), loss, k); b = -1 for priors.
    tags: factor index -> names of the edges it stands for (coverage)."""
    name: str
    poses: np.ndarray
    factors: list
    tags: dict = field(default_factory=dict)

    def tag(self, idx, *names):
        self.tags.setdefault(idx, set()).update(names)


def _spd(rng, cond, scale=1.0):
    Q, _ = np.linalg.qr(rng.standard_normal((3, 3)))
    ev = np.geomspace(1.0, 1.0 / cond, 3) * scale
    W = (Q * ev) @ Q.T
    return ((W + W.T) / 2).reshape(9)


def _rel(pa, pb):
    ca, sa = math.cos(pa[2]), math.sin(pa[2])
    dx, dy = pb[0] - pa[0], pb[1] - pa[1]
    return np.array([ca * dx + sa * dy, -sa * dx + ca * dy, pb[2] - pa[2]])


def headings(seed=11) -> Graph:
    """Headings 0, +-pi/2, +-pi, +-nextafter(pi, 0) on every pair in both orders; z[2] on the seam exactly, a few ulp
    off it, on +-(2j+1)pi up to ~300 rad, and away from it; priors on the same headings."""
    rng = np.random.default_rng(seed)
    pi_ = math.pi
    th = [0.0, pi_ / 2, -pi_ / 2, pi_, -pi_, math.nextafter(pi_, 0.0), -math.nextafter(pi_, 0.0)]
    poses = np.array([[0.5 * i, 0.25 * (i % 3), t] for i, t in enumerate(th)])
    g = Graph("headings", poses, [])
    W = _spd(rng, 1e3, 10.0)
    for a in range(len(th)):
        for b in range(len(th)):
            if a == b:
                continue
            d = th[b] - th[a]
            zxy = _rel(poses[a], poses[b])[:2] + rng.uniform(-0.1, 0.1, 2)
            zs = [d + pi_, d - pi_, math.nextafter(d + pi_, 9.0), math.nextafter(d - pi_, -9.0),
                  d + pi_ + 3 * 2 ** -51, d + 0.3]
            j = int(rng.integers(0, 48))
            zs.append(d + (2 * j + 1) * pi_)
            zs.append(d - (2 * j + 1) * pi_)
            for z2 in zs:
                g.factors.append((1, a, b, np.array([zxy[0], zxy[1], z2]), W, 0, 0.0))
                g.tag(len(g.factors) - 1, "heading", "a<b" if a < b else "a>b")
    for a in range(len(th)):
        for z2 in (th[a] + pi_, th[a] - pi_, math.nextafter(th[a] + pi_, 9.0), th[a] + 95 * pi_, th[a] - 0.2):
            g.factors.append((2, a, -1, np.array([poses[a, 0] + 0.01, poses[a, 1], z2]), W, 0, 0.0))
            g.tag(len(g.factors) - 1, "prior_heading")
    return g


def coordinates(seed=12) -> Graph:
    """|x|, |y| up to 1e9 with separations 1e-3 ... 1e3 (cancellation in dx, dy), W up to cond 1e12 and scaled by
    2^e, e in {-500, -100, 0, 100, 500}."""
    rng = np.random.default_rng(seed)
    poses, factors = [], []
    g = Graph("coordinates", None, factors)
    for base in (0.0, 1e3, 1e6, 1e9):
        for sep in (1e-3, 1.0, 1e3):
            for e in (-500, -100, 0, 100, 500):
                cond = float(rng.choice([1.0, 1e6, 1e12]))
                sgn = rng.choice([-1.0, 1.0], 2)
                pa = np.array([sgn[0] * base * rng.uniform(0.5, 1), sgn[1] * base * rng.uniform(0.5, 1),
                               rng.uniform(-math.pi, math.pi)])
                ang = rng.uniform(-math.pi, math.pi)
                pb = pa + np.array([sep * math.cos(ang), sep * math.sin(ang), rng.uniform(-1, 1)])
                a = len(poses)
                poses += [pa, pb]
                z = _rel(pa, pb) + rng.normal(0, 0.05, 3)
                W = _spd(rng, cond, 2.0 ** e)
                factors.append((1, a, a + 1, z, W, 0, 0.0))
                g.tag(len(factors) - 1, "coord", f"W2^{e}")
                factors.append((1, a + 1, a, -z, W, 0, 0.0))
                g.tag(len(factors) - 1, "coord", f"W2^{e}")
                factors.append((2, a, -1, pa + rng.normal(0, 1e-3, 3), W, 0, 0.0))
    g.poses = np.array(poses)
    return g


def losses(nan_rows=True) -> Graph:
    """The isolated loss cases of loss_rows(), each on its own pair of coincident poses (r = (r0, 0, 0) exactly).
    nan_rows=False leaves out the rows where W_eff was NaN before the loss was made total (Cauchy, k^2 = 0, s = 0):
    a solver fed them would be asked to factor a NaN system."""
    poses, factors = [], []
    g = Graph("losses", None, factors)
    for loss, k, r0, W00 in loss_rows():
        if not nan_rows and loss == CAUCHY and k * k == 0.0 and loss_s(r0, W00) == 0.0:
            continue
        p = np.array([3.0 + len(poses), -1.0, 0.0])
        a = len(poses)
        poses += [p, p.copy()]
        W = np.diag([W00, 1.0, 1.0]).reshape(9)
        factors.append((32, a, a + 1, np.array([r0, 0.0, 0.0]), W, loss, k))
        g.tag(len(factors) - 1, "loss", f"{'huber' if loss == HUBER else 'cauchy'}:{loss_band(k, loss_s(r0, W00))}")
        if r0 == 1.0 and W00 in straddle(k):
            with mpmath.workdps(DPS):
                side = "below" if mpmath.mpf(W00) <= mpmath.mpf(k) ** 2 else "above"
            g.tag(len(factors) - 1, f"{'huber' if loss == HUBER else 'cauchy'}:straddle_{side}")
    g.poses = np.array(poses)
    return g


def shapes(seed=13) -> Graph:
    """Kernel shapes: a hub pose with 80 incident factors, half with the hub as a and half as b, listed across warp
    boundaries; one pose pair with 44 parallel factors in both orientations; 37 further pairs (more than 32 dirty
    slots), N not a multiple of 4.  Robust factors with moderate k are mixed in."""
    rng = np.random.default_rng(seed)
    n_spokes, n_par, n_extra = 80, 44, 37
    N = 1 + n_spokes + 2 + 2 * n_extra
    N += (N % 4 == 0)
    poses = np.c_[rng.uniform(-50, 50, (N, 2)), rng.uniform(-math.pi, math.pi, N)]
    g = Graph("shapes", poses, [])
    Ws = [_spd(rng, c, s) for c, s in ((1.0, 100.0), (1e4, 10.0), (1e8, 1e3))]

    def add(ftype, a, b, loss=0, k=0.0, *tags):
        z = (_rel(poses[a], poses[b]) if b >= 0 else poses[a].copy()) + rng.normal(0, 0.2, 3)
        g.factors.append((ftype, a, b, z, Ws[len(g.factors) % 3], loss, k))
        g.tag(len(g.factors) - 1, *tags)

    for i in range(n_spokes):
        o = 1 + i
        loss = (HUBER, CAUCHY, 0)[i % 3]
        add(32 if loss else 1, 0, o, loss, 0.5, "hub") if i % 2 else add(32 if loss else 1, o, 0, loss, 0.5, "hub")
    p, q = n_spokes + 1, n_spokes + 2
    for i in range(n_par):
        loss = (0, CAUCHY)[i % 2]
        add(32 if loss else 1, p, q, loss, 2.0, "parallel") if i % 3 else add(32 if loss else 1, q, p, loss, 2.0,
                                                                               "parallel")
    for i in range(n_extra):
        a, b = n_spokes + 3 + 2 * i, n_spokes + 4 + 2 * i
        add(1, a, b) if i % 2 else add(1, b, a)
        add(1, a, 0)
    for a in range(N):
        add(2, a, -1)
    return g


def corpus(nan_rows=True) -> list:
    return [headings(), coordinates(), losses(nan_rows), shapes()]


def graph_refs(g: Graph, pts=None, node2q=None):
    """factor_ref of every factor of g, at the poses (or at pts (F, 6): a's point then b's), with the elimination order
    node2q (default: node id order)."""
    out = []
    for i, (t, a, b, z, W, loss, k) in enumerate(g.factors):
        pa = g.poses[a] if pts is None else pts[i, :3]
        pb = None if b < 0 else (g.poses[b] if pts is None else pts[i, 3:])
        early = b < 0 or (a < b if node2q is None else node2q[a] < node2q[b])
        out.append(factor_ref(t, z, W, pa, pb, loss, k, a_early=early, a_lower=b < 0 or a < b))
    return out
