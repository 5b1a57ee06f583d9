"""High-precision reference of the clover construction and the clover force with a per-element bound on the kernels'
rounding error (test-only, numpy).  The companion of tests/precise.py for the kernel families of clover_build.h
(clover_build_kernel, clover_invert_kernel, clover_trlog_kernel) and clover_force.h (clover_hop_force_kernel,
clover_sigma_kernel, clover_deriv_kernel).

The flat checks of tests/test_*_clover_build.py and clover_force_cases.deviation divide by the largest entry of the whole
field: in fp32 they cannot tell A from the identity on smooth links (A - 1 ~ eps is below 1e-5 there), and they cannot
see an error at a site whose spinors are small.  Here every element is checked against its own bound.

The reference reads exactly the values the kernel reads (fp64 or fp32 links, spinors after the native rotation, packed
A, mom) and computes in long double for fp64 kernels and in float64 for fp32 kernels, so the only difference between
kernel and reference is the kernel's own arithmetic.  Every real component must satisfy

    |got - ref| <= sqrt2 gamma_K T + E_in + u_P |ref|

with gamma_K = K u / (1 - K u) (Higham, Accuracy and Stability of Numerical Algorithms, 2nd ed., 3.1), u the unit
roundoff of the kernel's arithmetic, T the same computation on absolute values (complex moduli, so that one complex
product's real part |ar br| + |ai bi| is <= |a| |b|), E_in the propagated error of an earlier stage and u_P |ref| the
output rounding (precise.out_bound).  The sqrt2: the per-part error of a stage becomes a complex-modulus error when the
next stage multiplies it.  The constants are read off the site code, which uses explicit fma_rn / mul_rn (counts are
roundings along the longest chain a term passes through):

* `K_BUILD` = 42 for A = 1 + k S, k = coeff / 8.  A 3x3 complex product rounds each real output in a chain of 6 fused
  multiply-adds; a leaf is 3 products (18) and the four leaves accumulate into one q, so the first leaf's terms pass
  3 more chains (18); G = Q - Q^+ (1); S1 sums 2 planes and S2 4 planes of G (3, the first onto zero is exact); k S
  (1); k itself is coeff * 0.125 rounded to the field's precision (1).  The diagonal 1 -+ k S1 adds one rounding of
  the stored value, the output term.
* Inverse: A^-1 from the kernel's own A by Cholesky in double for fp64 and fp32 fields, checked normwise per chiral
  block: `K_CHOL` u_d kappa_2 ||A^-1||_2 (precise.K_CHOL; the explicit inverse M^+ M, M = L^-1, adds forward
  substitution and a product whose errors are of the same form, gamma_n |M| |L| and gamma_n |M^+| |M|), plus the
  rounding to the field's precision.
* tr log A per parity, first order: the Cholesky backward error |dA| <= 4 gamma_{n+1} |L| |L^+| (x 4 for complex
  arithmetic, as K_CHOL) moves log det by tr(A^-1 dA) <= 4 gamma_{n+1} sum_ij |A^-1|_ij (|L| |L^+|)_ji per block;
  every 2 log L_jj carries the sqrt rounding (u) and the double log (1 ulp, 2 u |log L_jj|); the sum is fixed-order
  (inst_clover_build.cu): 6 terms per block, 2 blocks per site, a 128-leaf tree per CTA (7), a strided serial sum of
  ceil(nblk / 128) CTA partials per thread and one more 128-leaf tree (7), so `trlog_depth` = 21 + ceil(nblk / 128)
  roundings times sum |2 log L_jj|.
* Force: `K_HOPF` = 16 + 2n for the hopping force U_mu(x) r: the spin projection (1), the spin trace as a chain of 8
  fmas per component, the fma accumulation of 2n traces into r (2n), force_coeff rounded to the field's precision (1),
  U r (6).  `K_SIGMA` = 12 + n for oprod: the spin trace (8), n fma accumulations, eps rounded (1), R - R^+ (1), the
  fma that adds the trace term (1).  `K_TRACE` = 5 for c tr[sigma A^-1]: a signed sum of 4 entries of A^-1 (3),
  sigma_coeff rounded (1), the fma into oprod (1); A^-1 enters with its normwise bound and its rounding to the field's
  precision.  `K_DERIV` = 48 for the insertion of oprod into the two leaves of each of the 3 planes holding U_mu(x):
  the backward recursion Y_j = l_j Y_{j+1} + O_j S_j puts the innermost insertion through 7 product chains of 6 (42)
  and the 6 leaves are summed into f (6); the oprod bound propagates through the |U| chains of the insertions.
  `K_TA` = 9 for mom -= TA(f) (mom_sub_ta), with the magnitudes |mom| + 2 |f|: the longest chain is the diagonal's
  trace / 3, difference, mean / 3 and final subtraction; an error in f reaches a mom component with a weight of at
  most 16/9 < 2, and an error already in mom passes the next projection with a weight of at most 4/3.  The hopping
  force and the derivative are projected and subtracted separately (two calls of mom_sub_ta), and so is their bound.
"""
import numpy as np

import clover_build_ref as R
import clover_force_ref as CF
import precise as PR
from quda_b200 import fields as F

K_BUILD, K_TRACE, K_DERIV, K_TA = 42, 5, 48, 9
U_D = 2.0 ** -53
SQ2 = PR.SQ2
BLOCK = 128  # threads per CTA of the trlog partial sums (kCloverBuildThreads)


def k_hopf(n):
    return 16 + 2 * n


def k_sigma(n):
    return 12 + n


def gamma(k, u):
    return k * u / (1 - k * u)


def trlog_depth(Vh):
    nblk = -(-Vh // BLOCK)
    return 21 + -(-nblk // BLOCK)


# ---------------------------------------------------------------------------------------------- helpers
def links(gauge, X, prec):
    """QDP gauge (the values the kernel reads) -> U[mu][t][z][y][x][3][3] in the reference precision"""
    g = np.asarray(gauge).astype(PR.real_t(prec))
    return np.stack([R.to_lex((g[mu, ..., 0] + 1j * g[mu, ..., 1]).astype(PR.cplx_t(prec)), X) for mu in range(4)])


def unpack(packed, prec):
    """packed [...][36] -> Hermitian [...][6][6] in the reference precision"""
    p = np.asarray(packed).astype(PR.real_t(prec))
    H = np.zeros(p.shape[:-1] + (6, 6), PR.cplx_t(prec))
    for i in range(6):
        H[..., i, i] = p[..., i]
    for n, (i, j) in enumerate(R.LOWER):
        H[..., i, j] = p[..., 6 + 2 * n] + 1j * p[..., 7 + 2 * n]
        H[..., j, i] = p[..., 6 + 2 * n] - 1j * p[..., 7 + 2 * n]
    return H


def pack(H):
    out = np.empty(H.shape[:-2] + (36,), H.real.dtype)
    out[..., 0:6] = np.real(np.diagonal(H, axis1=-2, axis2=-1))
    for n, (i, j) in enumerate(R.LOWER):
        out[..., 6 + 2 * n], out[..., 7 + 2 * n] = H[..., i, j].real, H[..., i, j].imag
    return out


def leaf_sum(U, mu, nu):
    """Q = sum of the four clover leaves at x (field_strength_tensor.cuh order); on |U| it is the leaves' T"""
    Um, Un = U[mu], U[nu]
    s = lambda a, dm, dn: R.shift(R.shift(a, mu, dm), nu, dn)  # noqa: E731
    Q = Um @ s(Un, 1, 0) @ R.dag(s(Um, 0, 1)) @ R.dag(Un)
    Q = Q + Un @ R.dag(s(Um, -1, 1)) @ R.dag(s(Un, -1, 0)) @ s(Um, -1, 0)
    Q = Q + R.dag(s(Un, 0, -1)) @ s(Um, 0, -1) @ s(Un, 1, -1) @ R.dag(Um)
    return Q + R.dag(s(Um, -1, 0)) @ R.dag(s(Un, -1, -1)) @ s(Um, -1, -1) @ s(Un, 0, -1)


def blocks(b1, b2, one):
    """chiral blocks [..][2][6][6] from b1[ch] (3x3, diagonal and lower used) and b2[ch] (the lower-left 3x3), the
    mapping of clover_build_ref.blocks_from_F"""
    shape = b1[0].shape[:-2]
    H = np.zeros(shape + (2, 6, 6), np.result_type(b1[0], b2[0], np.complex64))
    for ch in range(2):
        A = np.zeros(shape + (6, 6), H.dtype)
        for i in range(3):
            A[..., i, i] = one - b1[ch][..., i, i].real
            A[..., i + 3, i + 3] = one + b1[ch][..., i, i].real
        for (i, j) in [(1, 0), (2, 0), (2, 1)]:
            A[..., i, j] = -b1[ch][..., i, j]
            A[..., i + 3, j + 3] = b1[ch][..., i, j]
        A[..., 3:6, 0:3] = b2[ch]
        H[..., ch, :, :] = np.tril(A) + R.dag(np.tril(A, -1))
    return H


def planes(gauge, X, prec, leaf=leaf_sum):
    """(G = Q - Q^+ per plane, its T = |Q| + |Q|^T) on the lexicographic lattice"""
    U = links(gauge, X, prec)
    aU = np.abs(U).astype(np.float64)
    G, TG = [], []
    for mu, nu in R.PLANES:
        Q, Qa = leaf(U, mu, nu), leaf(aU, mu, nu)
        G.append(Q - R.dag(Q))
        TG.append(Qa + np.swapaxes(Qa, -1, -2))
    return G, TG


def build_from_planes(G, TG, X, coeff, prec):
    rt = PR.real_t(prec)
    k = rt(coeff) / rt(8)
    I = 1j
    b1 = [I * k * (G[0] - G[5]), I * k * (G[0] + G[5])]
    b2 = [k * (G[1] + G[4] - I * (G[2] - G[3])), k * (G[1] - G[4] - I * (G[2] + G[3]))]
    ref = R.from_lex(pack(blocks(b1, b2, rt(1))), X)
    ak = abs(float(k))
    t1 = ak * (TG[0] + TG[5])
    t2 = ak * (TG[1] + TG[4] + TG[2] + TG[3])
    T = np.abs(R.from_lex(pack(blocks([t1, t1], [t2, t2], 0.0)), X))
    T[..., 6:] = np.maximum(T[..., 6:], np.repeat(np.maximum(T[..., 6::2], T[..., 7::2]), 2, axis=-1))  # re and im alike
    return PR.Result(ref, SQ2 * gamma(K_BUILD, PR.U_P[prec]) * T)


# ---------------------------------------------------------------------------------------------- the clover construction
def clover_build(gauge, X, coeff, prec):
    """packed A [V][2][36] of the periodic lattice X from the QDP links the kernel reads, and its bound"""
    G, TG = planes(gauge, X, prec)
    return build_from_planes(G, TG, X, coeff, prec)


class Inverse:
    """A^-1 of the kernel's own packed A (reference precision), its Cholesky factor and the per-block data of the
    bounds: kappa_2 and ||A^-1||_2 [V][2]"""

    def __init__(self, packed, prec):
        self.prec = prec
        self.H = unpack(packed, 8)  # the kernel factors in double whatever the field's precision: long double here
        self.L = PR.cholesky(self.H)
        self.Hi = PR.hermitian_inverse(self.H)
        w = np.linalg.eigvalsh(self.H.astype(np.complex128))
        assert np.all(w[..., 0] > 0), "A is not positive definite"
        self.kappa = w[..., -1] / w[..., 0]
        self.norm_inv = 1.0 / w[..., 0]
        self.err = PR.K_CHOL * U_D * self.kappa * self.norm_inv  # normwise, per block

    def result(self):
        return PR.Result(pack(self.Hi), np.broadcast_to(self.err[..., None], self.Hi.shape[:-2] + (36,)).copy())

    def trlog(self, X):
        """Result of tr log A per parity ([2]; the kernel sums in double whatever the field's precision)"""
        n, u = 6, U_D
        d = np.real(np.diagonal(self.L, axis1=-2, axis2=-1))
        terms = 2 * np.log(d)                                   # [V][2][6]
        Vh = F.volume_cb(X)
        aL = np.abs(self.L).astype(np.float64)
        LL = aL @ np.swapaxes(aL, -1, -2)
        chol = 4 * gamma(n + 1, u) * np.einsum("...ij,...ji->...", np.abs(self.Hi).astype(np.float64), LL)
        aterm = np.abs(terms).astype(np.float64).sum(-1)
        per_block = chol + n * u + 2 * u * aterm
        depth = trlog_depth(Vh)
        ref, bound = [], []
        for p in range(2):
            sl = slice(p * Vh, (p + 1) * Vh)
            ref.append(terms[sl].sum())
            bound.append(per_block[sl].sum() + gamma(depth, u) * aterm[sl].sum())
        return PR.Result(np.array(ref), np.array(bound))


# ---------------------------------------------------------------------------------------------- the clover force
ONE4 = np.eye(4)


def outer_abs(a, b):
    return np.einsum("...sj,...sk->...jk", a, b)


def hop(U, aU, xs, ps, fc, prec):
    """(U_mu(x) r for every mu [4][lex][3][3], T [4][lex][3][3])"""
    rt = PR.real_t(prec)
    f = CF.hop_force(U, xs, ps, [rt(c) for c in fc])
    T = []
    for mu in range(4):
        Pp, Pm = np.abs(ONE4 + CF.GAMMA[mu]), np.abs(ONE4 - CF.GAMMA[mu])
        r = 0
        for x, p, c in zip(xs, ps, fc):
            ax, ap = np.abs(x).astype(np.float64), np.abs(p).astype(np.float64)
            r = r + abs(c) * (outer_abs(CF.spin(Pp, R.shift(ax, mu, 1)), ap) + outer_abs(CF.spin(Pm, R.shift(ap, mu, 1)), ax))
        T.append(aU[mu] @ r)
    return f, np.stack(T)


# the quadrants of the chiral blocks of A^-1 in tr[sigma A^-1], per plane (clover_trace.cuh)
_DIAG_QUADRANTS = (0, 5)


def sigma_trace(Hi, err, coeff, parity, X, prec):
    """(coeff tr[sigma A^-1] [6][lex][3][3] on the sites of `parity`, T, E: the propagated bound of A^-1)"""
    I = 1j
    UL, LR, UR, LL = Hi[..., :3, :3], Hi[..., 3:, 3:], Hi[..., :3, 3:], Hi[..., 3:, :3]
    mats = [I * (LR[:, 0] + LR[:, 1] - UL[:, 0] - UL[:, 1]), UR[:, 0] - LL[:, 0] + UR[:, 1] - LL[:, 1],
            -I * (UR[:, 0] + LL[:, 0] + UR[:, 1] + LL[:, 1]), I * (UR[:, 0] + LL[:, 0] - UR[:, 1] - LL[:, 1]),
            UR[:, 0] - LL[:, 0] - UR[:, 1] + LL[:, 1], I * (UL[:, 0] - LR[:, 0] - UL[:, 1] + LR[:, 1])]
    a = np.abs(Hi).astype(np.float64)
    aUL, aLR, aUR, aLL = a[..., :3, :3], a[..., 3:, 3:], a[..., :3, 3:], a[..., 3:, :3]
    mask = (CF.parity_lex(X) == parity)[..., None, None]
    rt = PR.real_t(prec)
    c, ac = rt(coeff), abs(coeff)
    E_site = 2 * (err[:, 0] + err[:, 1])[:, None, None] * np.ones((1, 3, 3))
    out, T, E = [], [], []
    for p, m in enumerate(mats):
        t = (aUL + aLR if p in _DIAG_QUADRANTS else aUR + aLL).sum(axis=1)
        out.append(np.where(mask, c * R.to_lex(m, X), 0))
        T.append(np.where(mask, ac * R.to_lex(t, X), 0))
        E.append(np.where(mask, ac * R.to_lex(E_site, X), 0))
    T = np.stack(T)
    return np.stack(out), T, np.stack(E) + PR.U_P[prec] * T


def sigma_oprod(xs, ps, eps, X, prec):
    """(R - R^+ [6][lex][3][3], T)"""
    rt = PR.real_t(prec)
    O = CF.sigma_oprod(xs, ps, [(rt(e[0]), rt(e[1])) for e in eps], X)
    par = CF.parity_lex(X)
    T = []
    for mu, nu in R.PLANES:
        r = 0
        for x, p, e in zip(xs, ps, eps):
            w = np.where(par == 0, abs(e[0]), abs(e[1]))[..., None, None]
            ax, ap = np.abs(x).astype(np.float64), np.abs(p).astype(np.float64)
            r = r + w * outer_abs(CF.spin(np.abs(CF.sigma(nu, mu)), ax), ap)
        T.append(r + np.swapaxes(r, -1, -2))
    return O, np.stack(T)


def deriv(U, O, absolute=False):
    """the insertions of O into the two leaves holding U_mu(x), summed over nu != mu (clover_force_ref.deriv); with
    `absolute` every term enters with + (U, O: absolute values)"""
    out = []
    for mu in range(4):
        f = 0
        for nu in range(4):
            if nu == mu:
                continue
            Ot = O[R.PLANES.index((max(mu, nu), min(mu, nu)))]
            s = lambda a, dm, dn: R.shift(R.shift(a, mu, dm), nu, dn)  # noqa: E731
            U1, U2, U3, U4 = U[mu], s(U[nu], 1, 0), s(U[mu], 0, 1), U[nu]
            up = (U1 @ U2 @ R.dag(U3) @ R.dag(U4) @ Ot + U1 @ U2 @ s(Ot, 1, 1) @ R.dag(U3) @ R.dag(U4)
                  + U1 @ U2 @ R.dag(U3) @ s(Ot, 0, 1) @ R.dag(U4) + U1 @ s(Ot, 1, 0) @ U2 @ R.dag(U3) @ R.dag(U4))
            L1, L2, L3, L4 = s(U[nu], 0, -1), s(U[mu], 0, -1), s(U[nu], 1, -1), U[mu]
            lo = (R.dag(L1) @ L2 @ s(Ot, 1, -1) @ L3 @ R.dag(L4) + Ot @ R.dag(L1) @ L2 @ L3 @ R.dag(L4)
                  + R.dag(L1) @ L2 @ L3 @ s(Ot, 1, 0) @ R.dag(L4) + R.dag(L1) @ s(Ot, 0, -1) @ L2 @ L3 @ R.dag(L4))
            sg = 1.0 if absolute or nu > mu else -1.0
            f = f + sg * up + (1.0 if absolute else -sg) * lo
        out.append(f)
    return np.stack(out)


def mom_sub_ta(m, f):
    """mom_sub_ta of clover_force.h in exact arithmetic: m [..][10] reals, f [..][3][3]"""
    m = m.copy()
    for n, (i, j) in enumerate(CF.OD):
        m[..., 2 * n] -= (f[..., i, j].real - f[..., j, i].real) * 0.5
        m[..., 2 * n + 1] -= (f[..., i, j].imag + f[..., j, i].imag) * 0.5
    tr = (f[..., 0, 0].imag + f[..., 1, 1].imag + f[..., 2, 2].imag) / 3
    d = m[..., 6:9] - (np.diagonal(f, axis1=-2, axis2=-1).imag - tr[..., None])
    m[..., 6:9] = d - d.mean(-1, keepdims=True)
    return m


def _per_link(a, X):
    """[4][lex][3][3] -> [V][4] maxima over the link's entries (parity-major sites)"""
    return np.stack([R.from_lex(a[mu], X).reshape(-1, 9).max(-1) for mu in range(4)], axis=1)


def _ta_step(m0, f, E, X, u):
    """(mom after one mom_sub_ta, bound on its error per link [V][4])"""
    fs = np.stack([R.from_lex(f[mu], X) for mu in range(4)], axis=1)
    m1 = mom_sub_ta(m0, fs)
    E_link = _per_link(E, X)
    F_link = _per_link(np.abs(f).astype(np.float64), X) + SQ2 * E_link
    M = np.maximum(np.abs(m0[..., :9]).max(-1), np.abs(m1[..., :9]).max(-1)).astype(np.float64)
    return m1, 2 * E_link + gamma(K_TA, u) * (M + 2 * F_link)


class Force:
    """the reference of b200_clover_force_accumulate and its bound, per link and real component of mom [V][4][10]:
    inputs are the values the kernel reads (spinors: native-basis lexicographic [t][z][y][x][4][3])"""

    def __init__(self, gauge, packed, xs, ps, fc, eps, sigma_coeff, trlog_parity, mom, X, prec, inverse=None):
        rt, u, n = PR.real_t(prec), PR.U_P[prec], len(xs)
        U = links(gauge, X, prec)
        aU = np.abs(U).astype(np.float64)
        f_hop, T_hop = hop(U, aU, xs, ps, fc, prec)
        O, T_o = sigma_oprod(xs, ps, eps, X, prec)
        inv = inverse or Inverse(packed, prec)
        O_tr, T_tr, E_tr = sigma_trace(inv.Hi, inv.err, sigma_coeff, trlog_parity, X, prec)
        O = O + O_tr
        E_O = gamma(k_sigma(n), u) * T_o + gamma(K_TRACE, u) * T_tr + E_tr
        f_der = deriv(U, O)
        aO = np.abs(O).astype(np.float64) + SQ2 * E_O
        E_der = deriv(aU, SQ2 * gamma(K_DERIV, u) * aO + SQ2 * E_O, absolute=True)
        E_hop = SQ2 * gamma(k_hopf(n), u) * T_hop
        m0 = np.asarray(mom).astype(rt)
        m1, e1 = _ta_step(m0, f_hop, E_hop, X, u)
        m2, e2 = _ta_step(m1, f_der, E_der, X, u)
        bound = np.zeros(m2.shape)
        bound[..., :9] = (4.0 / 3.0 * e1 + e2)[..., None]
        m2[..., 9] = m0[..., 9]  # the pad is never written
        self.result = PR.Result(m2, bound)
        self.O, self.E_O, self.f_hop, self.f_der = O, E_O, f_hop, f_der
