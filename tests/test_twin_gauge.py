"""CPU tier of the gauge half of an HMC step, on the host twin (tests/gaugetwin), which runs the library's entry points and
site code: the force against the reference's own host code and the numpy restatement, the update against scipy's expm,
the momentum action and the plaquette; a finite difference of the Wilson + rectangle action pins the sign and the
normalisation of the force; gauge covariance; the boundary sign; every refusal; a pure-gauge leapfrog."""
import numpy as np
import pytest
import scipy.linalg

import clover_force_ref as CF
import gauge_cases as G
from gauge_twin import gauge_twin

TOL = {8: 1e-13, 4: 1e-5}


def twin():
    return G.Runner(gauge_twin(), "twin")


needs_ref = pytest.mark.skipif(not G.have_ref(), reason="oracle/_ref/libquda_gaugeref.so is not built (no reference tree)")


def _force_case(X, paths, field, prec):
    V = int(np.prod(X))
    gauge = G.FIELDS[field](X, 11)
    mom0 = G.random_mom(V, 5, 0.1)
    p, c = G.path_set(paths)
    want = G.ref_force(mom0, gauge, X, p, c, 0.2)
    got = twin().force(mom0, gauge, X, p, c, 0.2, prec)
    assert G.deviation(got, want, mom0) <= TOL[prec]


@needs_ref
@pytest.mark.parametrize("X", G.SHAPES)
@pytest.mark.parametrize("paths", G.PATH_SETS)
@pytest.mark.parametrize("field", sorted(G.FIELDS))
def test_twin_matches_reference_force(X, paths, field):
    _force_case(X, paths, field, 8)


@needs_ref
@pytest.mark.parametrize("X", G.SHAPES)
@pytest.mark.parametrize("field", sorted(G.FIELDS))
def test_twin_fp32_matches_reference_force(X, field):
    _force_case(X, "plaq+rect", field, 4)


@pytest.mark.parametrize("X", [(4, 4, 4, 4), (2, 4, 4, 6)])
@pytest.mark.parametrize("paths", G.PATH_SETS)
def test_twin_matches_restatement_force(X, paths):
    V = int(np.prod(X))
    gauge = G.haar_links(X, 3)
    mom0 = G.random_mom(V, 4, 0.1)
    p, c = G.path_set(paths)
    got = twin().force(mom0, gauge, X, p, c, 0.3)
    assert G.deviation(got, G.force(mom0, gauge, X, p, c, 0.3), mom0) <= 1e-13


@needs_ref
@pytest.mark.parametrize("prec", [8, 4])
def test_twin_matches_reference_mom_action(prec):
    X = (4, 6, 8, 10)
    mom = G.random_mom(int(np.prod(X)), 9).astype(np.float64 if prec == 8 else np.float32)
    got, want = twin().mom_action(mom, X, prec), G.ref_mom_action(mom)
    # the reference squares fp32 momenta in fp32; the library squares them in double
    assert abs(got - want) <= {8: 1e-12, 4: 1e-7}[prec] * np.abs(mom).sum() ** 1
    assert abs(got - G.mom_action(mom)) <= 1e-12 * np.abs(mom).sum()


def _expm_update(gauge, mom, dt, conj_mom=False):
    P = G.traceless_p(mom, conj_mom)  # [V][4][3][3]
    U = G.cplx(gauge)  # [4][V][3][3]
    E = np.array([[scipy.linalg.expm(dt * P[v, mu]) for v in range(P.shape[0])] for mu in range(4)])
    return G.to_qdp(E @ U), P


def _special_mom(V, kind, seed):
    """momenta whose spectra are the hard cases of the closed-form exponential"""
    rng = np.random.default_rng(seed)
    if kind == "zero":
        return np.zeros((V, 4, 10))
    if kind == "tiny":
        return G.random_mom(V, seed, 1e-9)
    if kind == "generic":
        return G.random_mom(V, seed, 1.0)
    if kind == "large":
        return G.random_mom(V, seed, 3.0)
    z = rng.normal(size=(V, 4, 3, 3)) + 1j * rng.normal(size=(V, 4, 3, 3))
    q, _ = np.linalg.qr(z)
    a = rng.uniform(-1.5, 1.5, size=(V, 4))
    if kind == "degenerate":  # two equal eigenvalues: w = 0
        ev = np.stack([a, a, -2 * a], -1)
    else:  # "c0_zero": eigenvalues (a, -a, 0), det P = 0
        ev = np.stack([a, -a, 0 * a], -1)
    P = np.einsum("...ij,...j,...kj->...ik", q, 1j * ev, q.conj())
    return CF.mom_from_matrices(P)


@pytest.mark.parametrize("kind", ["zero", "tiny", "generic", "large", "degenerate", "c0_zero"])
@pytest.mark.parametrize("conj_mom", [False, True])
def test_twin_update_matches_expm(kind, conj_mom):
    X = (4, 4, 2, 2)
    V = int(np.prod(X))
    gauge = G.haar_links(X, 21)
    mom = _special_mom(V, kind, 22)
    dt = 0.7
    want, P = _expm_update(gauge, mom, dt, conj_mom)
    got = twin().update(gauge, mom, X, dt, conj_mom, exact=True)
    assert np.abs(got - want).max() <= 1e-14 * max(1.0, np.abs(dt * P).max() ** 2)
    if kind == "zero":
        assert np.array_equal(got, gauge)
    got8 = twin().update(gauge, mom, X, dt, conj_mom, exact=False)
    n = np.linalg.norm(dt * P, ord=2, axis=(-2, -1)).max()
    bound = n ** 9 / 362880 * np.exp(n) + 1e-14 * max(1.0, n ** 8)  # remainder of the order-8 Taylor series, |U| = 1
    assert np.abs(got8 - want).max() <= bound


def test_twin_update_fp32():
    X = (4, 4, 2, 2)
    gauge = G.haar_links(X, 23)
    mom = G.random_mom(int(np.prod(X)), 24)
    want, _ = _expm_update(gauge, mom, 0.3)
    assert np.abs(twin().update(gauge, mom, X, 0.3, exact=True, prec=4) - want).max() <= 2e-6
    want8 = twin().update(gauge, mom, X, 0.3, exact=False)  # the order-8 truncation is larger than fp32 rounding here
    assert np.abs(twin().update(gauge, mom, X, 0.3, exact=False, prec=4) - want8).max() <= 2e-6


@pytest.mark.parametrize("X", G.SHAPES)
@pytest.mark.parametrize("prec", [8, 4])
def test_twin_plaquette_matches_restatement(X, prec):
    gauge = G.haar_links(X, 31) if X[0] != 4 else G.near_identity_links(X, 31, 0.3)
    got, want = twin().plaquette(gauge, X, prec), G.plaquette(gauge, X)
    assert np.allclose(got, want, rtol=0, atol={8: 1e-14, 4: 1e-6}[prec])
    assert got[0] == 0.5 * (got[1] + got[2])


def test_finite_difference_pins_force_normalisation():
    """gauge_force with the Wilson + rectangle coefficients (c0 beta, c1 beta as path coefficients, eb3 = dt beta / 3 with
    the beta folded into the coefficients here) is dt times the derivative of the action along U -> exp(eps H) U, in the
    convention of test_twin_clover_force.py: sum_links tr(H F) = dS/d eps, F = (mom_after - mom_before) / dt"""
    X = (4, 4, 4, 6)
    V = int(np.prod(X))
    beta, c0, c1, dt = 2.3, 5.0 / 3, -1.0 / 12, 0.4
    gauge = G.near_identity_links(X, 41, 0.4)
    p, _ = G.path_set("plaq+rect")
    coeffs = [c0] * 6 + [c1] * 18
    mom0 = G.random_mom(V, 42, 0.5)
    mom1 = twin().force(mom0, gauge, X, p, coeffs, dt * beta / 3)
    Fm = CF.mom_to_matrices(mom1 - mom0) / dt  # [V][4][3][3]
    rng = np.random.default_rng(43)
    H = CF.ta(rng.normal(size=(4, V, 3, 3)) + 1j * rng.normal(size=(4, V, 3, 3)))
    predicted = np.einsum("mvij,vmji->", H, Fm).real
    eps = 1e-4
    U = G.cplx(gauge)
    S = {k: G.loop_action(G.to_qdp(G.expm_ah(k * eps * H) @ U), X, p, coeffs, beta) for k in (2, 1, -1, -2)}
    fd = (8 * (S[1] - S[-1]) - (S[2] - S[-2])) / (12 * eps)
    assert abs(fd - predicted) <= 1e-8 * abs(fd), (fd, predicted)


def test_force_is_gauge_covariant():
    """TA(U_mu(x) sum path) -> g(x) TA(...) g(x)^+ under U_mu(x) -> g(x) U_mu(x) g(x + mu)^+"""
    X = (4, 4, 4, 4)
    V = int(np.prod(X))
    import clover_build_ref as R
    gauge = G.haar_links(X, 51)
    g = G.cplx(G.haar_links(X, 52))[0]  # one SU(3) matrix per site, parity-major
    gl = R.to_lex(g, X)
    U = R.links(gauge, X)
    Ug = np.stack([gl @ U[mu] @ R.dag(R.shift(gl, mu, 1)) for mu in range(4)])
    gauge_g = G.to_qdp(np.stack([R.from_lex(Ug[mu], X) for mu in range(4)]))
    p, c = G.path_set("symanzik48")
    zero = np.zeros((V, 4, 10))
    F = CF.mom_to_matrices(twin().force(zero, gauge, X, p, c, 1.0))
    Fg = CF.mom_to_matrices(twin().force(zero, gauge_g, X, p, c, 1.0))
    rot = np.einsum("vab,vmbc,vdc->vmad", g, F, g.conj())
    assert np.abs(Fg - rot).max() <= 1e-13 * np.abs(F).max()


def test_boundary_sign_cancels():
    """force and plaquette bit-identical with and without the antiperiodic sign baked into the links; the update carries
    it: exp(dt P) (-U) = -(exp(dt P) U) exactly"""
    X = (4, 4, 4, 6)
    V = int(np.prod(X))
    gauge = G.haar_links(X, 61)
    signed = G.antiperiodic(gauge, X)
    assert not np.array_equal(gauge, signed)
    mom0 = G.random_mom(V, 62, 0.2)
    t = twin()
    for paths in G.PATH_SETS:
        p, c = G.path_set(paths)
        assert np.array_equal(t.force(mom0, gauge, X, p, c, 0.3), t.force(mom0, signed, X, p, c, 0.3))
    assert t.plaquette(gauge, X) == t.plaquette(signed, X)
    for exact in (True, False):
        a = t.update(gauge, mom0, X, 0.5, exact=exact)
        assert np.array_equal(G.antiperiodic(a, X), t.update(signed, mom0, X, 0.5, exact=exact))


def _force_args():
    X = (4, 4, 4, 4)
    V = int(np.prod(X))
    p, c = G.path_set("plaq")
    from quda_b200 import gauge as GP
    table, lengths, n, max_length = GP.path_table(p)
    return X, np.zeros((V, 4, 10)), G.near_identity_links(X, 1), table, lengths, c, n, max_length


@pytest.mark.parametrize("what", ["precision", "num_paths_0", "num_paths_over", "length_0", "length_over_max",
                                  "max_length_over", "step_8", "step_negative", "open_path"])
def test_force_refusals(what):
    from quda_b200 import lib as L
    X, mom, gauge, table, lengths, c, n, max_length = _force_args()
    prec = 2 if what == "precision" else 8
    if what == "num_paths_0":
        n = 0
    if what == "num_paths_over":
        reps = L.GAUGE_MAX_PATHS // n + 1
        table, lengths, c = np.concatenate([table] * reps, 1), lengths * reps, c * reps
        n = len(lengths)
    if what == "length_0":
        lengths = [0] + lengths[1:]
    if what == "length_over_max":
        lengths = [max_length + 1] + lengths[1:]
    if what == "max_length_over":
        max_length = L.GAUGE_MAX_LENGTH + 1
        table = np.pad(table, ((0, 0), (0, 0), (0, max_length - table.shape[2])))
    if what in ("step_8", "step_negative"):
        table = table.copy()
        table[2, 3, 1] = 8 if what == "step_8" else -1
    if what == "open_path":
        table = table.copy()
        table[1, 0, 2] = table[1, 0, 0]  # U_nu twice: ends at x + 2 nu-hat
    rc, out = twin().force_rc(mom, gauge, X, table, lengths, c, n, max_length, 0.1, prec)
    assert rc == -1  # B200_ERR_INVALID
    assert not out.any()


def test_force_table_limits_accepted():
    """the largest table the parameter block holds: B200_GAUGE_MAX_PATHS paths in rows of B200_GAUGE_MAX_LENGTH steps.  A
    closed loop has an even number of links, so the longest path in a row has B200_GAUGE_MAX_LENGTH - 1 steps (a 5 x 1
    rectangle)"""
    from quda_b200 import lib as L
    X = (4, 4, 4, 4)
    V = int(np.prod(X))
    k = L.GAUGE_MAX_LENGTH // 2 - 2
    loops = [[[mu + 1] * (1 + k) + [(mu + 1) % 4 + 1] + [-(mu + 1)] * (1 + k) + [-((mu + 1) % 4 + 1)]] * L.GAUGE_MAX_PATHS
             for mu in range(4)]
    p = G._paths(loops)
    assert len(p[0][0]) == L.GAUGE_MAX_LENGTH - 1
    coeffs = [1.0 / L.GAUGE_MAX_PATHS] * L.GAUGE_MAX_PATHS
    from quda_b200 import gauge as GP
    table, lengths, n, _ = GP.path_table(p)
    table = np.pad(table, ((0, 0), (0, 0), (0, 1)))
    gauge = G.near_identity_links(X, 71, 0.2)
    mom0 = G.random_mom(V, 72, 0.1)
    rc, got = twin().force_rc(mom0, gauge, X, table, lengths, coeffs, n, L.GAUGE_MAX_LENGTH, 0.5, 8)
    assert rc == 0
    assert G.deviation(got, G.force(mom0, gauge, X, p, coeffs, 0.5), mom0) <= 1e-13


@pytest.mark.parametrize("fn", ["update", "mom_action", "plaquette"])
def test_other_refusals(fn):
    import ctypes as C
    lib = gauge_twin()
    X = (C.c_int * 4)(4, 4, 4, 4)
    buf = np.zeros(64)
    q = (C.c_void_p * 4)(*[buf.ctypes.data] * 4)
    if fn == "update":
        assert lib.twin_update_gauge(q, q, buf.ctypes.data, X, 2, 0.1, 0, 1, None) == -1
        assert lib.twin_update_gauge(q, q, buf.ctypes.data, X, 8, float("nan"), 0, 1, None) == -1
        assert lib.twin_update_gauge(q, q, buf.ctypes.data, (C.c_int * 4)(4, 4, 3, 4), 8, 0.1, 0, 1, None) == -1
    elif fn == "mom_action":
        S = C.c_double()
        assert lib.twin_mom_action(C.byref(S), buf.ctypes.data, X, 2, None) == -1
        assert lib.twin_mom_action(None, buf.ctypes.data, X, 8, None) == -1
    else:
        p = (C.c_double * 3)()
        assert lib.twin_plaquette(p, q, X, 16, None) == -1
        assert lib.twin_plaquette(p, (C.c_void_p * 4)(buf.ctypes.data, None, None, None), X, 8, None) == -1


def _leapfrog(t, gauge, mom, X, paths, coeffs, beta, n, tau):
    dt = tau / n
    mom = t.force(mom, gauge, X, paths, coeffs, 0.5 * dt * beta / 3)
    for i in range(n):
        gauge = t.update(gauge, mom, X, dt)
        mom = t.force(mom, gauge, X, paths, coeffs, (dt if i < n - 1 else 0.5 * dt) * beta / 3)
    return gauge, mom


def test_pure_gauge_leapfrog():
    """Wilson gauge HMC on the twin: |dH| falls about 4x per halving of dt, and forward, negate P, back returns the links"""
    X = (4, 4, 4, 4)
    V = int(np.prod(X))
    beta, tau = 2.0, 1.0
    p, c = G.path_set("plaq")
    t = twin()
    gauge = G.near_identity_links(X, 81, 0.3)
    mom = G.random_mom(V, 82)

    def H(g, m):
        return t.mom_action(m, X) + beta * 6 * V * (1 - t.plaquette(g, X)[0])

    H0 = H(gauge, mom)
    dH = []
    for n in (16, 32, 64):
        g1, m1 = _leapfrog(t, gauge, mom, X, p, c, beta, n, tau)
        dH.append(abs(H(g1, m1) - H0))
    for a, b in zip(dH, dH[1:]):
        assert 3.0 <= a / b <= 5.0, dH
    g1, m1 = _leapfrog(t, gauge, mom, X, p, c, beta, 16, tau)
    g2, m2 = _leapfrog(t, g1, -m1, X, p, c, beta, 16, tau)
    assert np.abs(g2 - gauge).max() <= 1e-12
    assert np.abs(-m2 - mom).max() <= 1e-11
