"""TEST ORACLE of the clover construction, in numpy complex128: clover-leaf field strength, the chiral-block mapping of
the clover term, its inverse and log det.  The reference has no host implementation of this, so it is restated here from
the formulas of include/kernels/field_strength_tensor.cuh:40-178 (leaves, F = (Q - Q^dagger) / 8, no trace subtraction),
include/kernels/clover_compute.cuh:60-124 (blocks) and include/kernels/clover_invert.cuh:44-84 (inverse, tr log).

Field orders are the oracle's (oracle/__init__.py): QDP gauge [4][V][3][3][2] and packed clover [V][2][36] (6 real
diagonals + 15 complex strictly-lower entries, column-major), sites parity-major.  Internally every field is a
lexicographic array [t][z][y][x] so that a shift along dimension d is np.roll on axis 3 - d."""
import numpy as np

from quda_b200 import fields as F

PLANES = [(1, 0), (2, 0), (2, 1), (3, 0), (3, 1), (3, 2)]  # F10, F20, F21, F30, F31, F32
LOWER = [(i, j) for j in range(6) for i in range(j + 1, 6)]  # packed order of the strictly-lower entries


def _site_maps(X):
    """lexicographic index of every packed site (parity-major: parity * Vh + x_cb)"""
    idx = []
    for p in range(2):
        c = F.cb_coords(X, p)
        idx.append(((c[:, 3] * X[2] + c[:, 2]) * X[1] + c[:, 1]) * X[0] + c[:, 0])
    return np.concatenate(idx)


def to_lex(field_sites, X):
    """[V parity-major][...] -> [t][z][y][x][...]"""
    lex = np.empty_like(field_sites)
    lex[_site_maps(X)] = field_sites
    return lex.reshape((X[3], X[2], X[1], X[0]) + field_sites.shape[1:])


def from_lex(lex, X):
    V = X[0] * X[1] * X[2] * X[3]
    flat = lex.reshape((V,) + lex.shape[4:])
    return flat[_site_maps(X)]


def links(gauge, X):
    """QDP gauge -> complex U[mu][t][z][y][x][3][3]"""
    g = np.asarray(gauge, dtype=np.float64)
    c = g[..., 0] + 1j * g[..., 1]
    return np.stack([to_lex(c[mu], X) for mu in range(4)])


def shift(a, d, n):
    """a(x + n d)"""
    return np.roll(a, -n, axis=3 - d)


def dag(m):
    return np.conj(np.swapaxes(m, -1, -2))


def field_strength(U, mu, nu):
    """F_mu,nu = (Q - Q^dagger) / 8, Q the sum of the four clover leaves at x"""
    Um, Un = U[mu], U[nu]
    s = lambda a, dm, dn: shift(shift(a, mu, dm), nu, dn)  # noqa: E731  a(x + dm mu + dn nu)
    Q = Um @ s(Un, 1, 0) @ dag(s(Um, 0, 1)) @ dag(Un)
    Q = Q + Un @ dag(s(Um, -1, 1)) @ dag(s(Un, -1, 0)) @ s(Um, -1, 0)
    Q = Q + dag(s(Un, 0, -1)) @ s(Um, 0, -1) @ s(Un, 1, -1) @ dag(Um)
    Q = Q + dag(s(Um, -1, 0)) @ dag(s(Un, -1, -1)) @ s(Um, -1, -1) @ s(Un, 0, -1)
    return (Q - dag(Q)) / 8.0


def blocks_from_F(Fs, coeff):
    """the two 6x6 chiral blocks of A per site, [...][2][6][6], from the six planes (clover_compute.cuh:82-121 without the
    factor 1/2 of the native storage)"""
    I = 1j
    b1 = [I * coeff * (Fs[0] - Fs[5]), I * coeff * (Fs[0] + Fs[5])]
    b2 = [coeff * (Fs[1] + Fs[4] - I * (Fs[2] - Fs[3])), coeff * (Fs[1] - Fs[4] - I * (Fs[2] + Fs[3]))]
    shape = Fs[0].shape[:-2]
    H = np.zeros(shape + (2, 6, 6), dtype=np.complex128)
    for ch in range(2):
        A = np.zeros(shape + (6, 6), dtype=np.complex128)
        for i in range(3):
            A[..., i, i] = 1.0 - b1[ch][..., i, i].real
            A[..., i + 3, i + 3] = 1.0 + b1[ch][..., i, i].real
        for (i, j) in [(1, 0), (2, 0), (2, 1)]:
            A[..., i, j] = -b1[ch][..., i, j]
            A[..., i + 3, j + 3] = b1[ch][..., i, j]
        A[..., 3:6, 0:3] = b2[ch]
        # Hermitian: the upper triangle mirrors the lower one
        A = np.tril(A) + dag(np.tril(A, -1))
        H[..., ch, :, :] = A
    return H


def pack(H):
    """[...][2][6][6] Hermitian -> packed [...][2][36]"""
    out = np.empty(H.shape[:-2] + (36,), dtype=np.float64)
    out[..., 0:6] = np.real(np.diagonal(H, axis1=-2, axis2=-1))
    for n, (i, j) in enumerate(LOWER):
        out[..., 6 + 2 * n] = H[..., i, j].real
        out[..., 7 + 2 * n] = H[..., i, j].imag
    return out


def unpack(packed):
    """packed [...][36] -> Hermitian [...][6][6]"""
    p = np.asarray(packed, dtype=np.float64)
    H = np.zeros(p.shape[:-1] + (6, 6), dtype=np.complex128)
    for i in range(6):
        H[..., i, i] = p[..., i]
    for n, (i, j) in enumerate(LOWER):
        H[..., i, j] = p[..., 6 + 2 * n] + 1j * p[..., 7 + 2 * n]
        H[..., j, i] = p[..., 6 + 2 * n] - 1j * p[..., 7 + 2 * n]
    return H


def all_planes(gauge, X):
    """[6][t][z][y][x][3][3]: F10, F20, F21, F30, F31, F32"""
    U = links(gauge, X)
    return np.stack([field_strength(U, mu, nu) for mu, nu in PLANES])


def compute_clover(gauge, X, coeff):
    """packed A [V][2][36] (float64) of the QDP gauge field on the periodic lattice X"""
    Fs = all_planes(gauge, X)
    return from_lex(pack(blocks_from_F(list(Fs), coeff)), X)


def invert(packed):
    """(A^-1 packed, log det per block [V][2])"""
    H = unpack(packed)
    sign, logdet = np.linalg.slogdet(H)
    assert np.all(sign.real > 0)
    return pack(np.linalg.inv(H)), logdet


def trlog(packed):
    """sum of log det A over the sites of each parity (both chiral blocks)"""
    _, ld = invert(packed)
    Vh = ld.shape[0] // 2
    return np.array([ld[:Vh].sum(), ld[Vh:].sum()])
