"""Extended-precision reference of the five-point essential-matrix problem (mpmath, 60 digits), independent of the fp64 solver it
checks (oracle/hv_oracle_essential.c and csrc/essential.cu):

  1. the exact doubles q (5 x 4: x1, y1, x2, y2, normalised) become mpf; the null space of the 5 x 9 epipolar matrix (row i:
     x2_a x1_b for E[a][b]) is the last four columns of the orthogonal factor of mpmath's own QR: E = x X + y Y + z Z + W;
  2. the ten cubic constraints det E = 0 and 2 E E^T E - tr(E E^T) E = 0 are expanded symbolically (polynomials as dicts of exponents);
  3. elimination by the hidden variable z (Li and Hartley, "Five-point motion estimation made easy", ICPR 2006): the constraints are
     C(z) m(x, y) = 0 over the ten monomials of x, y up to degree 3, and det C(z) has degree 10 (column degrees 0, 0, 0, 0, 1, 1, 1, 2,
     2, 3). Its coefficients come from C(z)'s determinant at eleven Chebyshev nodes, interpolated at 80 digits;
  4. all ten roots from mp.polyroots; a root is real when its imaginary part is below 1e-30 of its magnitude. The number of real roots
     is checked against a Sturm sequence of the same polynomial;
  5. per real root, (x, y) from C(z)'s null vector (the monomial 1 fixed at 1, the other nine by least squares), E normalised to unit
     Frobenius norm;
  6. per solution the componentwise condition number kappa with respect to q, from the implicit-function derivative: on the solution,
     F(E, q) = (the five epipolar residuals, the ten constraints, |E|^2 - 1) = 0 has full column rank in E, so dE/dq = -J_E^+ J_q.
     kappa = max over the entries of E of sum_j |dE/dq_j| |q_j|: a relative change u of every q_j moves E by at most about kappa u;
  7. per set, whether its number of real roots is fp64-determined: the same count (Sturm) for a few seeded draws of q with every entry
     moved by up to 4 ulp.
Self-checks (raise AssertionError): every reference E satisfies the constraints and the five epipolar equations to 1e-40; polyroots
and the Sturm count agree; det C(z) has no coefficient past degree 10 (checked at a twelfth node)."""
import numpy as np
from mpmath import mp

DPS = 60                 # digits of the roots, the solutions and kappa
FORM_DPS = 80            # digits of the null space, the constraints and the interpolation of det C(z)
REAL_CUT = 30            # a root is real when |Im| < 10^-REAL_CUT |root|
CHECK_TOL = 40           # self-checks: constraints and epipolar equations below 10^-CHECK_TOL
PERTURB_ULP = 4
PERTURB_DRAWS = 3

# monomials of x, y up to degree 3 (exponents); the last is 1
XY = [(3, 0), (2, 1), (1, 2), (0, 3), (2, 0), (1, 1), (0, 2), (1, 0), (0, 1), (0, 0)]


def _padd(a, b, s=1):
    out = dict(a)
    for k, v in b.items():
        out[k] = out.get(k, 0) + s * v
    return out


def _pmul(a, b):
    out = {}
    for ka, va in a.items():
        for kb, vb in b.items():
            k = (ka[0] + kb[0], ka[1] + kb[1], ka[2] + kb[2])
            out[k] = out.get(k, 0) + va * vb
    return out


def _pscale(a, s):
    return {k: v * s for k, v in a.items()}


def _mpq(q):
    return [[mp.mpf(float(v)) for v in row] for row in np.asarray(q, np.float64)]


def _null_basis(Q):
    """X, Y, Z, W (each 9 entries, E row-major) spanning the null space of the epipolar matrix"""
    A = mp.matrix(9, 5)
    for i, (x1, y1, x2, y2) in enumerate(Q):
        a, b = (x2, y2, mp.mpf(1)), (x1, y1, mp.mpf(1))
        for r in range(3):
            for c in range(3):
                A[3 * r + c, i] = a[r] * b[c]
    O, _ = mp.qr(A, mode="full")
    return [[O[k, 5 + c] for k in range(9)] for c in range(4)]


def _constraints(N):
    """the ten cubic constraints as polynomials {(i, j, k): coefficient of x^i y^j z^k}"""
    E = [[{(1, 0, 0): N[0][3 * r + c], (0, 1, 0): N[1][3 * r + c], (0, 0, 1): N[2][3 * r + c], (0, 0, 0): N[3][3 * r + c]}
          for c in range(3)] for r in range(3)]
    EEt = [[None] * 3 for _ in range(3)]
    for a in range(3):
        for b in range(a, 3):
            s = {}
            for c in range(3):
                s = _padd(s, _pmul(E[a][c], E[b][c]))
            EEt[a][b] = EEt[b][a] = s
    tr = _padd(_padd(EEt[0][0], EEt[1][1]), EEt[2][2])
    out = []
    minor = [_padd(_pmul(E[1][1], E[2][2]), _pmul(E[1][2], E[2][1]), -1),
             _padd(_pmul(E[1][2], E[2][0]), _pmul(E[1][0], E[2][2]), -1),
             _padd(_pmul(E[1][0], E[2][1]), _pmul(E[1][1], E[2][0]), -1)]
    det = {}
    for c in range(3):
        det = _padd(det, _pmul(E[0][c], minor[c]))
    out.append(det)
    for a in range(3):
        for b in range(3):
            s = {}
            for c in range(3):
                s = _padd(s, _pmul(EEt[a][c], E[c][b]))
            out.append(_padd(_pscale(s, 2), _pmul(tr, E[a][b]), -1))
    return out


def _hidden(cons):
    """C[e][m]: the coefficients (ascending powers of z, 4 entries) of monomial XY[m] in constraint e"""
    C = [[[mp.mpf(0)] * 4 for _ in XY] for _ in cons]
    col = {xy: m for m, xy in enumerate(XY)}
    for e, p in enumerate(cons):
        for (i, j, k), v in p.items():
            C[e][col[(i, j)]][k] += v
    return C


def _det(M):
    """determinant by Gaussian elimination with partial pivoting (M is consumed)"""
    n, d = len(M), mp.mpf(1)
    for k in range(n):
        p = max(range(k, n), key=lambda r: abs(M[r][k]))
        if M[p][k] == 0:
            return mp.mpf(0)
        if p != k:
            M[k], M[p] = M[p], M[k]
            d = -d
        d *= M[k][k]
        for r in range(k + 1, n):
            f = M[r][k] / M[k][k]
            if f:
                Mr, Mk = M[r], M[k]
                for c in range(k + 1, n):
                    Mr[c] -= f * Mk[c]
    return d


def _Cz(C, z):
    return [[((row[m][3] * z + row[m][2]) * z + row[m][1]) * z + row[m][0] for m in range(10)] for row in C]


_VINV = {}


def _poly(C):
    """ascending coefficients of det C(z) (degree 10) from eleven Chebyshev nodes; a twelfth node checks the degree"""
    if mp.prec not in _VINV:
        nodes = [mp.cos(mp.pi * (2 * k + 1) / 22) for k in range(11)]
        _VINV[mp.prec] = (nodes, mp.inverse(mp.matrix([[t ** k for k in range(11)] for t in nodes])))
    nodes, Vinv = _VINV[mp.prec]
    vals = [_det(_Cz(C, t)) for t in nodes]
    coef = [mp.fsum(Vinv[k, i] * vals[i] for i in range(11)) for k in range(11)]
    t = mp.mpf("0.123456789")
    got, want = _det(_Cz(C, t)), mp.polyval(coef[::-1], t)
    scale = max(abs(v) for v in vals)
    assert abs(got - want) <= mp.mpf(10) ** (-FORM_DPS + 20) * scale, "det C(z) is not of degree 10"
    return coef


def _sturm_count(coef):
    """number of distinct real roots of the polynomial (ascending coefficients), by a Sturm sequence"""
    def trim(p):
        p = list(p)
        s = max(abs(v) for v in p)
        while len(p) > 1 and abs(p[-1]) <= s * mp.mpf(10) ** (-mp.dps + 10):
            p.pop()
        return p

    p0 = trim(coef)
    p1 = trim([k * coef[k] for k in range(1, len(p0))])
    seq = [p0, p1]
    while len(seq[-1]) > 1:
        a, b = list(seq[-2]), seq[-1]
        while len(a) >= len(b):
            f = a[-1] / b[-1]
            sh = len(a) - len(b)
            for i in range(len(b)):
                a[sh + i] -= f * b[i]
            a.pop()
        if not a or max(abs(v) for v in a) <= max(abs(v) for v in seq[-2]) * mp.mpf(10) ** (-mp.dps + 10):
            break
        seq.append([-v for v in trim(a)])

    def changes(signs):
        s = [v for v in signs if v != 0]
        return sum(1 for u, v in zip(s, s[1:]) if u != v)
    at_pos = [mp.sign(p[-1]) for p in seq]
    at_neg = [mp.sign(p[-1]) * (-1) ** (len(p) - 1) for p in seq]
    return changes(at_neg) - changes(at_pos)


def _form(q):
    """(null basis, hidden-variable matrix, ascending coefficients of det C(z)) at FORM_DPS"""
    with mp.workdps(FORM_DPS):
        Q = _mpq(q)
        N = _null_basis(Q)
        C = _hidden(_constraints(N))
        return Q, N, C, _poly(C)


def _xy(C, z):
    """(x, y) of root z: C(z)'s null vector with the monomial 1 fixed at 1, the other nine from the normal equations"""
    M = _Cz(C, z)
    A = mp.matrix([[M[e][m] for m in range(9)] for e in range(10)])
    b = mp.matrix([-M[e][9] for e in range(10)])
    v = mp.lu_solve(A.T * A, A.T * b)
    return v[7], v[8]


def _unit(N, x, y, z):
    E = [x * N[0][k] + y * N[1][k] + z * N[2][k] + N[3][k] for k in range(9)]
    n = mp.sqrt(mp.fsum(e * e for e in E))
    return [e / n for e in E]


def _residuals(E, Q):
    """max |constraint| and max |epipolar residual| of the unit E (9 entries, row-major)"""
    M = mp.matrix(3, 3)
    for k in range(9):
        M[k // 3, k % 3] = E[k]
    G = 2 * M * M.T * M - sum(M[i, j] ** 2 for i in range(3) for j in range(3)) * M
    con = max([abs(mp.det(M))] + [abs(G[i, j]) for i in range(3) for j in range(3)])
    ep = max(abs(mp.fsum((x2, y2, 1)[a] * M[a, b] * (x1, y1, 1)[b] for a in range(3) for b in range(3))) for x1, y1, x2, y2 in Q)
    return con, ep


def _kappa(E, Q):
    """componentwise condition number of the unit E with respect to q (implicit-function derivative)"""
    M = [[E[3 * a + b] for b in range(3)] for a in range(3)]
    rows_E, rows_q = [], []
    for i, (x1, y1, x2, y2) in enumerate(Q):
        a, b = (x2, y2, 1), (x1, y1, 1)
        rows_E.append([a[r] * b[c] for r in range(3) for c in range(3)])
        Ex1 = [mp.fsum(M[r][c] * b[c] for c in range(3)) for r in range(3)]
        x2E = [mp.fsum(a[r] * M[r][c] for r in range(3)) for c in range(3)]
        rq = [mp.mpf(0)] * 20
        rq[4 * i], rq[4 * i + 1], rq[4 * i + 2], rq[4 * i + 3] = x2E[0], x2E[1], Ex1[0], Ex1[1]
        rows_q.append(rq)
    # d det = sum cof * dE
    cof = [[M[(r + 1) % 3][(c + 1) % 3] * M[(r + 2) % 3][(c + 2) % 3] - M[(r + 1) % 3][(c + 2) % 3] * M[(r + 2) % 3][(c + 1) % 3]
            for c in range(3)] for r in range(3)]
    rows_E.append([cof[r][c] for r in range(3) for c in range(3)])
    # d (2 E E^T E - tr(E E^T) E) = 2 (dE E^T E + E dE^T E + E E^T dE) - 2 tr(E dE^T) E - tr(E E^T) dE
    EtE = [[mp.fsum(M[k][r] * M[k][c] for k in range(3)) for c in range(3)] for r in range(3)]
    EEt = [[mp.fsum(M[r][k] * M[c][k] for k in range(3)) for c in range(3)] for r in range(3)]
    tr = EEt[0][0] + EEt[1][1] + EEt[2][2]
    for a in range(3):
        for b in range(3):
            row = []
            for r in range(3):
                for c in range(3):       # derivative by E[r][c]
                    v = 0
                    if r == a:
                        v += 2 * EtE[c][b]
                    v += 2 * M[a][c] * M[r][b]
                    if c == b:
                        v += 2 * EEt[a][r]
                    v -= 2 * M[r][c] * M[a][b]
                    if r == a and c == b:
                        v -= tr
                    row.append(v)
            rows_E.append(row)
    rows_E.append([E[k] for k in range(9)])
    # dE/dq_j = -G^-1 J_E[i]^T dF_i/dq_j with G = J_E^T J_E: only epipolar row i = j // 4 depends on q_j
    G = mp.matrix([[mp.fsum(r[a] * r[b] for r in rows_E) for b in range(9)] for a in range(9)])
    H = [mp.lu_solve(G, mp.matrix(rows_E[i])) for i in range(5)]
    D = mp.matrix(9, 20)
    for j in range(20):
        for k in range(9):
            D[k, j] = -H[j // 4][k] * rows_q[j // 4][j]
    qv = [Q[i][j] for i in range(5) for j in range(4)]
    return max(mp.fsum(abs(D[k, j] * qv[j]) for j in range(20)) for k in range(9))


def _perturbed(q, rng):
    b = np.ascontiguousarray(q, np.float64).view(np.int64).copy()
    b += rng.integers(-PERTURB_ULP, PERTURB_ULP + 1, b.shape) * np.where(b >= 0, 1, -1)
    return b.view(np.float64)


def count_real(q):
    """the number of real roots of the set's degree-10 polynomial (Sturm)"""
    _, _, _, coef = _form(q)
    with mp.workdps(DPS):
        return _sturm_count([+c for c in coef])


def solve5(q, seed=0, determined=True):
    """The reference solutions of five normalised correspondences q (5, 4) float64: a dict with
    E (k, 3, 3) float64 (unit Frobenius norm, sign arbitrary), kappa (k,), z (k,) the hidden-variable roots, count k, and
    determined: the count is the same for PERTURB_DRAWS draws of q moved by up to PERTURB_ULP ulp per entry (None if not asked)."""
    Q, N, C, coef = _form(q)
    with mp.workdps(DPS):
        coef = [+c for c in coef]
        roots = mp.polyroots(coef[::-1], maxsteps=400, extraprec=4 * DPS)
        real = sorted(mp.re(r) for r in roots if abs(mp.im(r)) < mp.mpf(10) ** -REAL_CUT * abs(r))
        assert len(real) == _sturm_count(coef), "polyroots and the Sturm sequence disagree on the number of real roots"
        Es, kap = [], []
        tol = mp.mpf(10) ** -CHECK_TOL
        for z in real:
            x, y = _xy(C, z)
            E = _unit(N, x, y, z)
            con, ep = _residuals(E, Q)
            assert con < tol and ep < tol, f"reference solution z = {mp.nstr(z, 8)}: constraints {mp.nstr(con, 3)}, epipolar {mp.nstr(ep, 3)}"
            Es.append([float(e) for e in E])
            kap.append(float(_kappa(E, Q)))
    det = None
    if determined:
        rng = np.random.default_rng(seed)
        det = all(count_real(_perturbed(q, rng)) == len(real) for _ in range(PERTURB_DRAWS))
    return {"E": np.array(Es).reshape(-1, 3, 3), "kappa": np.array(kap), "z": np.array([float(z) for z in real]),
            "count": len(real), "determined": det}
