"""Extended-precision reference for the P3P problem (tests/test_pnp_ref.py): mpmath at 60 digits, sharing no code or formulation with
the solver (oracle/hv_oracle_pnp.c, csrc/pnp.cu).

Grunert's system: the distances s1, s2, s3 along the unit rays f1, f2, f3 satisfy si^2 + sj^2 - 2 si sj cij = dij^2. With u = s2 / s1
and v = s3 / s1 this is two conics in (u, v). Here u is eliminated by the Sylvester resultant of the two conics (as quadratics in u),
evaluated at 60 digits at five values of v and interpolated to the quartic in v; the solver instead writes u as a quotient of
polynomials in v and expands the quartic in closed form. The roots come from mp.polyroots, and their number on (0, inf) is checked
by a Sturm count. For each real v > 0, u is the common root of the two conics (the root of the first that the second vanishes at).
Solutions with u or v not positive are dropped. A solution is (s1, s2, s3).

fp64-determined: the number of solutions is the same for 8 perturbations of the inputs (world points and ray directions) by up to
4 ulp. kappa: the componentwise condition number of each solution with respect to those inputs, from forward differences at 60 digits."""
import mpmath as mp
import numpy as np

mp.mp.dps = 60


def rays(xy, fx, fy, cx, cy):
    """unit rays of float32 pixels (3, 2), exactly as the pixels and intrinsics are given"""
    out = []
    for u, v in np.asarray(xy, np.float64):
        x = (mp.mpf(float(u)) - mp.mpf(cx)) / mp.mpf(fx)
        y = (mp.mpf(float(v)) - mp.mpf(cy)) / mp.mpf(fy)
        n = mp.sqrt(x * x + y * y + 1)
        out.append([x / n, y / n, 1 / n])
    return out


def _dot(a, b):
    return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]


def _sub(a, b):
    return [a[0] - b[0], a[1] - b[1], a[2] - b[2]]


def _conics(X, f):
    c12, c13, c23 = _dot(f[0], f[1]), _dot(f[0], f[2]), _dot(f[1], f[2])
    d12, d13, d23 = (_dot(_sub(X[i], X[j]), _sub(X[i], X[j])) for i, j in ((0, 1), (0, 2), (1, 2)))

    # as quadratics in u with coefficients in v: (a2, a1, a0)
    def q1(v):
        return (d13, -2 * d13 * c12, d13 - d12 * (1 + v * v - 2 * v * c13))

    def q2(v):
        return (d23 - d12, -2 * d23 * c12 + 2 * d12 * v * c23, d23 - d12 * v * v)
    return q1, q2


def _resultant(a, b):
    """Sylvester resultant of a2 u^2 + a1 u + a0 and b2 u^2 + b1 u + b0"""
    S = mp.matrix([[a[0], a[1], a[2], 0], [0, a[0], a[1], a[2]], [b[0], b[1], b[2], 0], [0, b[0], b[1], b[2]]])
    return mp.det(S)


def quartic(X, f):
    """the resultant's coefficients (descending) in v, by interpolation at v = 0..4"""
    q1, q2 = _conics(X, f)
    nodes = [mp.mpf(k) for k in range(5)]
    vals = [_resultant(q1(v), q2(v)) for v in nodes]
    V = mp.matrix([[v ** (4 - j) for j in range(5)] for v in nodes])
    return list(mp.lu_solve(V, mp.matrix(vals)))


def sturm_count(c, lo, hi):
    """distinct real roots of the polynomial c (descending) in (lo, hi]"""
    def pdiv(a, b):
        a = list(a)
        q = []
        while len(a) >= len(b):
            k = a[0] / b[0]
            q.append(k)
            for i in range(len(b)):
                a[i] -= k * b[i]
            a.pop(0)
        return a

    def trim(p):
        while len(p) > 1 and abs(p[0]) < mp.mpf(10) ** (-40) * max(abs(x) for x in p):
            p = p[1:]
        return p
    seq = [trim(list(c)), trim([c[i] * (len(c) - 1 - i) for i in range(len(c) - 1)])]
    while len(seq[-1]) > 1 or abs(seq[-1][0]) > 0:
        r = pdiv(seq[-2], seq[-1])
        r = [-x for x in r]
        if not r or max(abs(x) for x in r) < mp.mpf(10) ** (-45) * max(abs(x) for x in seq[-2]):
            break
        seq.append(trim(r))
        if len(seq[-1]) == 1:
            break

    def changes(x):
        vals = [mp.polyval(p, x) for p in seq]
        vals = [v for v in vals if v != 0]
        return sum(1 for a, b in zip(vals, vals[1:]) if (a > 0) != (b > 0))
    return changes(lo) - changes(hi)


def solve(X, f):
    """every solution (s1, s2, s3) with positive depths, ascending in v; and the quartic's Sturm count on (0, inf)"""
    X = [[mp.mpf(float(c)) for c in p] for p in X]
    c = quartic(X, f)
    while abs(c[0]) == 0:
        c = c[1:]
    roots = mp.polyroots(c, maxsteps=400, extraprec=400)
    scale = max(abs(x) for x in c)
    R = 1 + max(abs(x / c[0]) for x in c[1:]) if len(c) > 1 else 1
    q1, q2 = _conics(X, f)
    d12 = _dot(_sub(X[0], X[1]), _sub(X[0], X[1]))
    c12 = _dot(f[0], f[1])
    sols = []
    for r in roots:
        if abs(mp.im(r)) > mp.mpf(10) ** (-30) * max(1, abs(r)):
            continue
        v = mp.re(r)
        if v <= 0:
            continue
        a, b = q1(v), q2(v)
        disc = a[1] * a[1] - 4 * a[0] * a[2]
        if disc < 0:
            disc = mp.mpf(0)
        cands = [(-a[1] + s * mp.sqrt(disc)) / (2 * a[0]) for s in (1, -1)]
        u = min(cands, key=lambda t: abs(b[0] * t * t + b[1] * t + b[2]))
        if u <= 0:
            continue
        s1 = mp.sqrt(d12 / (1 + u * u - 2 * u * c12))
        sols.append((v, [s1, u * s1, v * s1]))
    sols.sort(key=lambda t: t[0])
    del scale
    return [s for _, s in sols], sturm_count(c, mp.mpf(0), R)


def _perturbed(X, f, rng, ulps):
    Xp = [[mp.mpf(float(c)) * (1 + ulps * mp.mpf(2) ** -53 * rng.uniform(-1, 1)) for c in p] for p in X]
    fp = [[c * (1 + ulps * mp.mpf(2) ** -53 * rng.uniform(-1, 1)) for c in r] for r in f]
    return Xp, fp


def reference(X, xy, fx, fy, cx, cy, seed=0):
    """(solutions [(s1, s2, s3) as floats], sturm count, fp64-determined, kappa per solution)"""
    f = rays(xy, fx, fy, cx, cy)
    sols, sturm = solve(X, f)
    rng = np.random.default_rng(seed)
    determined = all(len(solve(*_perturbed(X, f, rng, 4))[0]) == len(sols) for _ in range(8))
    kappas = []
    if determined and sols:
        h = mp.mpf(10) ** -25
        base = np.array([[float(s) for s in sol] for sol in sols])
        grads = np.zeros((len(sols), 3))
        inputs = [("X", i, k) for i in range(3) for k in range(3)] + [("f", i, k) for i in range(3) for k in range(3)]
        for kind, i, k in inputs:
            Xp = [[mp.mpf(float(c)) for c in p] for p in X]
            fp = [list(r) for r in f]
            if kind == "X":
                x0 = Xp[i][k]
                Xp[i][k] = x0 * (1 + h) if x0 != 0 else h
            else:
                x0 = fp[i][k]
                fp[i][k] = x0 * (1 + h) if x0 != 0 else h
            sp, _ = solve(Xp, fp)
            if len(sp) != len(sols):
                return [[float(s) for s in sol] for sol in sols], sturm, False, []
            for j in range(len(sols)):
                grads[j] += np.abs([float((sp[j][q] - sols[j][q]) / h) for q in range(3)])
        kappas = list((grads / np.abs(base)).max(1))
    return [[float(s) for s in sol] for sol in sols], sturm, determined, kappas
