"""CPU tier: the clover term, its inverse and tr log A computed from the links by the host twin of the library's site code
(quda_b200/csrc/clover_build.h, built for the CPU by tests/clovertwin), against the numpy restatement
(tests/clover_build_ref.py) and against physics checks that do not use the restated block mapping; the argument checks of
b200_compute_clover / b200_clover_invert_packed; the depth-1 halo of comm.extend_gauge on 2 and 4 gloo ranks."""
import ctypes as C

import numpy as np
import pytest

import clover_build_ref as R
import oracle
from clover_twin import clover_twin
from dist_worker import run_ranks
from quda_b200 import dslash as D
from quda_b200 import fields as F
from quda_b200 import lib as L

LATTICES = [(4, 4, 4, 4), (4, 6, 2, 8)]
COEFFS = [0.12195 * 1.0, 0.13 * 1.9]
TOL = {8: 1e-13, 4: 1e-5}
NO_BORDER = (0, 0, 0, 0)

# DeGrand-Rossi gamma matrices (gamma_5 = gamma_1 gamma_2 gamma_3 gamma_4 = diag(1, 1, -1, -1)) and
# sigma_mu,nu = (i/2) [gamma_mu, gamma_nu]
_i = 1j
GAMMA = [np.array([[0, 0, 0, _i], [0, 0, _i, 0], [0, -_i, 0, 0], [-_i, 0, 0, 0]]),
         np.array([[0, 0, 0, -1], [0, 0, 1, 0], [0, 1, 0, 0], [-1, 0, 0, 0]]),
         np.array([[0, 0, _i, 0], [0, 0, 0, -_i], [-_i, 0, 0, 0], [0, _i, 0, 0]]),
         np.array([[0, 0, 1, 0], [0, 0, 0, 1], [1, 0, 0, 0], [0, 1, 0, 0]])]


def sigma(mu, nu):
    return 0.5j * (GAMMA[mu] @ GAMMA[nu] - GAMMA[nu] @ GAMMA[mu])


# With F = (Q - Q^dagger) / 8 anti-Hermitian, the reference's blocks (clover_compute.cuh) applied in the DeGrand-Rossi basis
# are A psi = psi + K coeff sum_{mu<nu} sigma_mu,nu F_mu,nu psi with K = i (fitted once against the reference's mapping,
# residual at rounding level).
K = 1j


def twin_clover(gauge, X, coeff, prec, border=NO_BORDER):
    out = np.zeros((int(np.prod(X)), 2, 36), dtype=oracle._dt(prec))
    D.compute_clover(out, gauge, X, border, prec, coeff, backend=clover_twin())
    return out


def twin_invert(packed, X, prec):
    inv = np.zeros_like(packed)
    return inv, D.clover_invert(inv, packed, X, prec, backend=clover_twin())


@pytest.mark.parametrize("X", LATTICES)
@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("coeff", COEFFS)
def test_twin_matches_reference(X, prec, coeff):
    gauge = oracle.random_gauge(X, prec, seed=11, antiperiodic_t=True)
    got = twin_clover(gauge, X, coeff, prec)
    want = R.compute_clover(gauge.astype(np.float64), X, coeff)
    assert np.abs(got - want).max() <= TOL[prec]
    assert F.clover_is_compressible(got, tol=1e-12 if prec == 8 else 1e-6)


@pytest.mark.parametrize("prec", [8, 4])
def test_unit_links_give_unit_clover(prec):
    X = (4, 4, 2, 6)
    gauge = np.zeros((4, int(np.prod(X)), 3, 3, 2), dtype=oracle._dt(prec))
    for c in range(3):
        gauge[:, :, c, c, 0] = 1.0
    got = twin_clover(gauge, X, 0.3, prec)
    want = np.zeros_like(got)
    want[..., 0:6] = 1.0
    assert np.array_equal(got, want)


@pytest.mark.parametrize("X", LATTICES)
def test_clover_is_one_plus_sigma_F(X):
    """oracle.apply_clover(A) psi == (1 + K coeff sum sigma F) psi with sigma from the DeGrand-Rossi gammas"""
    coeff = COEFFS[1]
    gauge = oracle.random_gauge(X, 8, seed=12)
    A = twin_clover(gauge, X, coeff, 8)
    Fsite = np.stack([R.from_lex(f, X) for f in R.all_planes(gauge, X)])  # [6][V][3][3]
    Vh = F.volume_cb(X)
    for p in range(2):
        psi = oracle.random_spinor(X, 8, seed=3 + p)
        c = psi[..., 0] + 1j * psi[..., 1]
        want = c.copy()
        for k, (mu, nu) in enumerate(R.PLANES):
            want += K * coeff * np.einsum("st,vab,vtb->vsa", sigma(mu, nu), Fsite[k][p * Vh:(p + 1) * Vh], c)
        got = oracle.apply_clover(A, psi, X, p)
        assert np.abs(got[..., 0] + 1j * got[..., 1] - want).max() < 1e-13


def test_gauge_covariance():
    """A[U^g] (g psi) == g (A[U] psi) for a random site-local SU(3) transform g, U^g_mu(x) = g(x) U_mu(x) g(x+mu)^dagger"""
    X, coeff = (4, 4, 4, 4), COEFFS[0]
    gauge = oracle.random_gauge(X, 8, seed=13)
    rng = np.random.default_rng(5)
    z = rng.normal(size=(int(np.prod(X)), 3, 3)) + 1j * rng.normal(size=(int(np.prod(X)), 3, 3))
    qm, r = np.linalg.qr(z)
    qm = qm * (np.diagonal(r, axis1=1, axis2=2) / np.abs(np.diagonal(r, axis1=1, axis2=2)))[:, None, :]
    g = qm / np.linalg.det(qm)[:, None, None] ** (1.0 / 3.0)  # SU(3), one per site (parity-major)
    U = gauge[..., 0] + 1j * gauge[..., 1]
    g_lex = R.to_lex(g, X)
    Ug = np.empty_like(U)
    for mu in range(4):
        u_lex = R.to_lex(U[mu], X)
        Ug[mu] = R.from_lex(g_lex @ u_lex @ R.dag(R.shift(g_lex, mu, 1)), X)
    gauge_g = np.stack([Ug.real, Ug.imag], axis=-1)
    A, Ag = twin_clover(gauge, X, coeff, 8), twin_clover(gauge_g, X, coeff, 8)
    Vh = F.volume_cb(X)
    for p in range(2):
        gp = g[p * Vh:(p + 1) * Vh]
        psi = oracle.random_spinor(X, 8, seed=21 + p)
        rot = lambda v: np.einsum("vab,vsb->vsa", gp, v[..., 0] + 1j * v[..., 1])  # noqa: E731
        lhs = oracle.apply_clover(Ag, np.stack([rot(psi).real, rot(psi).imag], axis=-1), X, p)
        rhs = rot(oracle.apply_clover(A, psi, X, p))
        assert np.abs(lhs[..., 0] + 1j * lhs[..., 1] - rhs).max() < 1e-13


@pytest.mark.parametrize("X", LATTICES)
@pytest.mark.parametrize("prec", [8, 4])
def test_inverse_and_trlog(X, prec):
    gauge = oracle.random_gauge(X, prec, seed=14)
    A = twin_clover(gauge, X, COEFFS[1], prec)
    inv, tl = twin_invert(A, X, prec)
    A64 = A.astype(np.float64)
    eye = np.broadcast_to(np.eye(6), (A.shape[0], 2, 6, 6))
    assert np.abs(R.unpack(A64) @ R.unpack(inv.astype(np.float64)) - eye).max() <= (1e-13 if prec == 8 else 1e-5)
    assert np.abs(inv - oracle.clover_invert(A)).max() <= TOL[prec]
    want_inv, _ = R.invert(A64)
    assert np.abs(inv - want_inv).max() <= TOL[prec]
    assert np.allclose(tl, R.trlog(A64), rtol=0, atol=1e-10)
    _, tl2 = twin_invert(A, X, prec)
    assert tl2 == tl  # fixed summation order: bit-identical
    tl3 = D.clover_invert(None, A, X, prec, backend=clover_twin())  # trlog only
    assert tl3 == tl


@pytest.mark.parametrize("world,grid_dims,Xl", [(2, (1, 1, 1, 2), (4, 4, 4, 4)), (4, (2, 1, 1, 2), (4, 4, 2, 4))])
def test_extend_gauge_matches_global_reference(world, grid_dims, Xl):
    """t split over 2 ranks; x and t split over 4 ranks (the corners of the x-t plane come from the diagonal neighbour)"""
    from clover_build_worker import worker
    clover_twin()  # build once in the parent
    for r in run_ranks(worker, world, (grid_dims, Xl, "host"), timeout=300):
        assert r["dev"] <= 1e-13, (r["rank"], r["dev"])
        assert np.allclose(r["trlog"], r["trlog_ref"], rtol=0, atol=1e-10), r


def _args(ptr=1):
    X = (C.c_int * 4)(4, 4, 4, 4)
    q = (C.c_void_p * 4)(ptr, ptr, ptr, ptr)
    return X, q, (C.c_int * 4)(0, 0, 0, 1)


@pytest.mark.parametrize("case", ["null_packed", "null_qdp", "null_link", "null_X", "null_border", "odd_X", "zero_X",
                                  "negative_X", "border_2", "border_neg", "prec_2", "prec_16", "coeff_nan", "coeff_inf"])
def test_compute_clover_refuses(case):
    lib = clover_twin().lib
    buf = np.zeros(16)
    X, q, b = _args(buf.ctypes.data)
    packed, prec, coeff, qa, Xa, ba = buf.ctypes.data, 8, 0.1, q, X, b
    if case == "null_packed":
        packed = None
    elif case == "null_qdp":
        qa = None
    elif case == "null_link":
        q[2] = None
    elif case == "null_X":
        Xa = None
    elif case == "null_border":
        ba = None
    elif case == "odd_X":
        X[1] = 5
    elif case == "zero_X":
        X[2] = 0
    elif case == "negative_X":
        X[3] = -4
    elif case == "border_2":
        b[0] = 2
    elif case == "border_neg":
        b[1] = -1
    elif case == "prec_2":
        prec = 2
    elif case == "prec_16":
        prec = 16
    elif case == "coeff_nan":
        coeff = float("nan")
    else:
        coeff = float("inf")
    assert lib.twin_compute_clover(packed, qa, Xa, ba, prec, coeff, None) == -1  # B200_ERR_INVALID
    assert b"b200_compute_clover" in lib.twin_last_error()


@pytest.mark.parametrize("case", ["null_packed", "null_trlog", "null_X", "odd_X", "zero_X", "prec_2"])
def test_clover_invert_refuses(case):
    lib = clover_twin().lib
    buf = np.zeros(16)
    X, _, _ = _args()
    tl = (C.c_double * 2)()
    packed, tla, Xa, prec = buf.ctypes.data, tl, X, 4
    if case == "null_packed":
        packed = None
    elif case == "null_trlog":
        tla = None
    elif case == "null_X":
        Xa = None
    elif case == "odd_X":
        X[0] = 3
    elif case == "zero_X":
        X[1] = 0
    else:
        prec = 2
    assert lib.twin_clover_invert_packed(None, tla, packed, Xa, prec, None) == -1
    assert b"b200_clover_invert_packed" in lib.twin_last_error()


def test_library_needs_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    lib = L.load()
    buf = np.zeros(16)
    X, q, b = _args(buf.ctypes.data)
    tl = (C.c_double * 2)()
    assert lib.b200_compute_clover(buf.ctypes.data, q, X, b, 8, 0.1, None) == -4  # B200_ERR_NO_DEVICE
    assert lib.b200_clover_invert_packed(None, tl, buf.ctypes.data, X, 8, None) == -4


def test_anisotropic_gauge_is_refused():
    with pytest.raises(L.B200Error, match="anisotropic"):
        D.compute_clover_field(np.zeros((4, 16, 3, 3, 2)), (2, 2, 2, 2), 8, 0.1, 1.0, anisotropy=2.0)


def test_clover_scale_matches_load_clover_formulas():
    """the (diagonal, max_element) helper both load_clover and compute_clover_field call, on numpy and torch inputs"""
    import torch
    c = oracle.random_clover((4, 4, 4, 4), 8, seed=3)
    for compressed in (True, False):
        d, m = D.clover_scale(c, compressed)
        _, meta = F.clover_to_native(c, (4, 4, 4, 4), 8, compressed=compressed)
        if compressed:
            assert abs(d - meta["diagonal"]) < 1e-15
        assert abs(m - meta["max_element"]) < 1e-15
        dt, mt = D.clover_scale(torch.from_numpy(c), compressed)
        assert abs(dt - d) < 1e-15 and abs(mt - m) < 1e-15
