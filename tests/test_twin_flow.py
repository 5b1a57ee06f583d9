"""CPU tier of the gradient flow and its observables, on the host twin (tests/flowtwin), which runs the site code and the
stage sequence of inst_gauge_flow.cu: against the numpy restatement tests/flow_ref.py, with the sign and normalisation of
the generator pinned by a finite difference of the action, the order of the integrator, closed forms on constant abelian
flux, the symmetries of E and Q, negative controls that each check must reject, and the argument checks."""
import ctypes as C

import numpy as np
import pytest

import flow_cases as FC
import flow_ref as FR
import gauge_cases as GC
from flow_twin import flow_twin
from quda_b200 import gauge as GP


def twin():
    return FC.Runner(flow_twin(), "twin")


def rel(a, b):
    return np.abs(np.asarray(a) - np.asarray(b)).max() / np.abs(np.asarray(b)).max()


# ------------------------------------------------------------------ 1. the restatement, fp32, one call against five
@pytest.mark.parametrize("X", FC.SHAPES)
@pytest.mark.parametrize("action", FC.ACTIONS)
@pytest.mark.parametrize("field", sorted(FC.FIELDS))
def test_twin_matches_restatement(X, action, field):
    gauge = FC.FIELDS[field](X, 7)
    paths, coeffs = GP.FLOW_ACTIONS[action]
    got = twin().flow(gauge, X, action)
    want = FR.flow(gauge, X, paths, coeffs, FC.EPS, FC.STEPS)
    assert np.abs(got - want).max() <= 1e-12
    e, q, dens = twin().observables(got, X)
    e_ref, q_ref, dens_ref = FR.observables(got, X)
    scale = np.abs(dens_ref).sum()
    assert rel(e, e_ref) <= 1e-12
    assert abs(q - q_ref) <= 1e-12 * scale and np.abs(dens - dens_ref).max() <= 1e-12 * np.abs(dens_ref).max()
    # fp32 against fp64
    got4 = twin().flow(gauge, X, action, prec=4)
    assert np.abs(got4 - got).max() <= 1e-5
    e4, q4, _ = twin().observables(got4.astype(np.float32), X, prec=4)
    assert rel(e4, e) <= 1e-5 and abs(q4 - q) <= 1e-5 * scale
    # five calls of one step: bit for bit
    step = gauge
    for _ in range(FC.STEPS):
        step = twin().flow(step, X, action, n_steps=1)
    assert np.array_equal(step, got)


# ------------------------------------------------------------------ 2. sign and normalisation
def _fd_and_norm(gauge, X, paths, coeffs, flow, h=1e-3):
    """(dS/dt at t = 0 by a five-point stencil of S(W_eps), -sum ||TA(Omega)||_F^2 from gauge_force and mom_action).  The
    stencil cancels the h^2 term of the plain central difference, which alone is larger than the tolerance; RK3's local
    error is even in eps and cancels too."""
    S = {k: FR.action(flow(gauge, k * h), X, paths, coeffs) for k in (2, 1, -1, -2)}
    fd = (8 * (S[1] - S[-1]) - (S[2] - S[-2])) / (12 * h)
    V = int(np.prod(X))
    m = GC.Runner(flow_twin(), "twin").force(np.zeros((V, 4, 10)), gauge, X, paths, coeffs, 1.0)  # -TA(Omega)
    norm2 = 2 * (GC.Runner(flow_twin(), "twin").mom_action(m, X) + 16 * V)
    return fd, -norm2


SYMANZIK_LOOPS = (GC.path_set("plaq+rect")[0], [5.0 / 3] * 6 + [-1.0 / 12] * 18)


@pytest.mark.parametrize("action", FC.ACTIONS)
@pytest.mark.parametrize("field", sorted(FC.FIELDS))
def test_finite_difference_pins_sign_and_normalisation(action, field):
    X = (4, 4, 4, 4)
    gauge = FC.FIELDS[field](X, 12)
    if action == "symanzik":
        paths, coeffs = SYMANZIK_LOOPS
        assert GP.FLOW_ACTIONS["symanzik"] == (paths, coeffs)
    else:
        paths, coeffs = GC.path_set("plaq")
        assert GP.FLOW_ACTIONS["wilson"] == (paths, coeffs)
    fd, want = _fd_and_norm(gauge, X, paths, coeffs, lambda g, e: twin().flow(g, X, action, eps=e, n_steps=1))
    print(action, field, "dS/dt", fd, "-sum |TA(Omega)|^2", want)
    assert abs(fd - want) <= 1e-8 * abs(want)


# ------------------------------------------------------------------ 3. order
def test_rk3_is_third_order():
    X, t = (4, 4, 4, 4), 0.2
    gauge = GC.near_identity_links(X, 21, 0.3)
    eps = 0.02
    ref = twin().flow(gauge, X, "wilson", eps=eps / 8, n_steps=80)
    errs = [np.abs(twin().flow(gauge, X, "wilson", eps=e, n_steps=round(t / e)) - ref).max() for e in (eps, eps / 2)]
    print("link errors at eps, eps/2:", errs, "ratio", errs[0] / errs[1])
    assert 6 <= errs[0] / errs[1] <= 10


# ------------------------------------------------------------------ 4. the Wilson flow lowers the Wilson action
def test_wilson_flow_raises_the_plaquette():
    X = (4, 6, 8, 10)
    g = GC.haar_links(X, 4)
    plaq = [twin().plaquette(g, X)[0]]
    for _ in range(20):
        g = twin().flow(g, X, "wilson", n_steps=1)
        plaq.append(twin().plaquette(g, X)[0])
    print("plaquette along the flow:", plaq)
    assert all(b > a for a, b in zip(plaq, plaq[1:]))


# ------------------------------------------------------------------ 5. constant abelian flux
@pytest.mark.parametrize("case", range(3))
@pytest.mark.parametrize("X", [(4, 6, 8, 10), (6, 6, 6, 6)])
def test_constant_abelian_flux(case, X):
    planes, sign = FC.flux_cases()[case]
    gauge, phis = FR.abelian_flux(X, planes)
    for action in FC.ACTIONS:
        assert np.abs(twin().flow(gauge, X, action) - gauge).max() <= 1e-14  # a stationary point of both actions
    e, q, _ = twin().observables(gauge, X)
    assert abs(e[0] - FC.flux_energy(phis)) <= 1e-13 * FC.flux_energy(phis)
    want = FC.flux_charge(phis, planes, sign)
    assert abs(q - want) <= 1e-12
    flipped = [[planes[0][0], -planes[0][1]], planes[1]]
    assert abs(twin().observables(FR.abelian_flux(X, flipped)[0], X)[1] + want) <= 1e-12
    # the restatement agrees (its charge is the one the negative control perturbs)
    assert abs(FR.observables(gauge, X)[1] - want) <= 1e-12


# ------------------------------------------------------------------ 6. symmetries
@pytest.mark.parametrize("action", FC.ACTIONS)
def test_gauge_invariance_and_covariance(action):
    X = (4, 6, 8, 10)
    gauge = GC.haar_links(X, 8)
    g = FR.random_su3((X[3], X[2], X[1], X[0]), 9)
    gauge2 = FR.gauge_transform(gauge, X, g)
    e, q, _ = twin().observables(gauge, X)
    e2, q2, dens = twin().observables(gauge2, X)
    assert rel(e2, e) <= 1e-12 and abs(q2 - q) <= 1e-12 * np.abs(dens).sum()
    assert rel(twin().plaquette(gauge2, X), twin().plaquette(gauge, X)) <= 1e-12
    f, f2 = twin().flow(gauge, X, action), twin().flow(gauge2, X, action)
    assert np.abs(f2 - FR.gauge_transform(f, X, g)).max() <= 1e-12


def test_reflection_flips_the_charge():
    X = (4, 6, 8, 10)
    gauge = twin().flow(GC.near_identity_links(X, 10, 0.6), X, "wilson")
    e, q, dens = twin().observables(gauge, X)
    e2, q2, _ = twin().observables(FR.reflect_x(gauge, X), X)
    print("Q", q, "reflected", q2)
    assert rel(e2, e) <= 1e-12 and abs(q2 + q) <= 1e-12 * np.abs(dens).sum() and abs(q) > 1e-3 * np.abs(dens).sum()


@pytest.mark.parametrize("action", FC.ACTIONS)
def test_boundary_sign_is_carried_bit_for_bit(action):
    X = (4, 6, 8, 10)
    gauge = GC.haar_links(X, 13)
    f = twin().flow(gauge, X, action)
    fa = twin().flow(GC.antiperiodic(gauge, X), X, action)
    assert np.array_equal(fa, GC.antiperiodic(f, X))
    assert twin().observables(fa, X)[:2] == twin().observables(f, X)[:2]


# ------------------------------------------------------------------ 7. negative controls
def test_euler_step_fails_the_restatement_check():
    X = (4, 4, 4, 4)
    gauge = GC.haar_links(X, 7)
    paths, coeffs = GP.FLOW_ACTIONS["wilson"]
    got = twin().flow(gauge, X, "wilson")
    euler = FR.flow(gauge, X, paths, coeffs, FC.EPS, FC.STEPS, step=FR.euler_step)
    assert np.abs(got - euler).max() > 1e-6


def test_flipped_generator_fails_the_finite_difference():
    X = (4, 4, 4, 4)
    gauge = GC.haar_links(X, 12)
    paths, coeffs = GP.FLOW_ACTIONS["wilson"]

    def flipped(g, e):
        return FR.flow(g, X, paths, coeffs, e, 1, step=lambda U, p, c, h: FR.euler_step(U, p, c, h, sign=-1.0))

    fd, want = _fd_and_norm(gauge, X, paths, coeffs, flipped)
    assert abs(fd - want) > 1.0 * abs(want)
    fd, want = _fd_and_norm(gauge, X, paths, coeffs, lambda g, e: FR.flow(g, X, paths, coeffs, e, 1, step=FR.euler_step))
    assert abs(fd - want) <= 1e-8 * abs(want)  # the unflipped Euler step passes: the control isolates the sign


def test_flipped_pairing_sign_fails_the_flux_check():
    X = (4, 6, 8, 10)
    planes, sign = FC.flux_cases()[2]  # flux in (0,3) and (1,2): the charge is tr F21 F30 alone
    gauge, phis = FR.abelian_flux(X, planes)
    bad = FR.observables(gauge, X, pair_signs=(1, -1, -1))[1]
    assert abs(bad - FC.flux_charge(phis, planes, sign)) > 1.0


# ------------------------------------------------------------------ 8. validation and bookkeeping
def test_refusals():
    X = (4, 4, 4, 4)
    V = int(np.prod(X))
    r = twin()
    paths, coeffs = GP.FLOW_ACTIONS["wilson"]
    table, lengths, n, ml = GP.path_table(paths)
    g = GC.haar_links(X, 1)
    for kw in ({"n_steps": 0}, {"n_steps": -1}, {"eps": np.nan}, {"eps": np.inf}):
        args = dict(eps=0.01, n_steps=1) | kw
        assert r.flow_rc(g, X, table, lengths, coeffs, n, ml, **args)[0] == -1
    bad = table.copy()
    bad[1, 2, 0] = 8  # out of range
    assert r.flow_rc(g, X, bad, lengths, coeffs, n, ml, 0.01, 1)[0] == -1
    bad = table.copy()
    bad[2, 0, 1] = (bad[2, 0, 1] + 1) % 4  # open
    assert r.flow_rc(g, X, bad, lengths, coeffs, n, ml, 0.01, 1)[0] == -1
    assert r.flow_rc(g, X, table, lengths, coeffs, 0, ml, 0.01, 1)[0] == -1
    lib = flow_twin()
    buf = np.zeros((4, V, 18))
    q = (C.c_void_p * 4)(*[buf[d].ctypes.data for d in range(4)])
    qn = (C.c_void_p * 4)(buf[0].ctypes.data, None, buf[2].ctypes.data, buf[3].ctypes.data)
    Xc = (C.c_int * 4)(*X)
    tp = table.ctypes.data_as(C.POINTER(C.c_int))
    L, Cf = (C.c_int * n)(*lengths), (C.c_double * n)(*coeffs)
    for out, inp, t, l, c in ((None, q, tp, L, Cf), (q, None, tp, L, Cf), (qn, q, tp, L, Cf), (q, qn, tp, L, Cf), (q, q, None, L, Cf),
                              (q, q, tp, None, Cf), (q, q, tp, L, None)):
        assert lib.twin_gauge_flow(out, inp, Xc, 8, t, l, c, n, ml, 0.01, 1, None) == -1
    assert lib.twin_gauge_flow(q, q, (C.c_int * 4)(4, 4, 4, 3), 8, tp, L, Cf, n, ml, 0.01, 1, None) == -1
    assert lib.twin_gauge_flow(q, q, Xc, 2, tp, L, Cf, n, ml, 0.01, 1, None) == -1
    e, qc = (C.c_double * 3)(), C.c_double()
    assert lib.twin_gauge_observables(None, C.byref(qc), None, q, Xc, 8, None) == -1
    assert lib.twin_gauge_observables(e, None, None, q, Xc, 8, None) == -1
    assert lib.twin_gauge_observables(e, C.byref(qc), None, qn, Xc, 8, None) == -1
    assert lib.twin_gauge_observables(e, C.byref(qc), None, None, Xc, 8, None) == -1
    assert lib.twin_gauge_observables(e, C.byref(qc), None, q, Xc, 4 + 4, None) == 0  # and NULL density is allowed


@pytest.mark.parametrize("X", [(4, 6, 8, 10), (6, 2, 4, 6)])
def test_density_sums_to_q_and_repeats(X):
    gauge = twin().flow(GC.haar_links(X, 2), X, "symanzik")
    e, q, dens = twin().observables(gauge, X)
    assert abs(dens.sum() - q) <= 1e-12 * np.abs(dens).sum()
    assert twin().observables(gauge, X)[:2] == (e, q)
    assert np.array_equal(twin().flow(gauge, X, "symanzik"), twin().flow(gauge, X, "symanzik"))
    # in place equals out of place, for an odd and an even number of steps (the ping-pong ends in either field)
    for n in (1, 2):
        assert np.array_equal(twin().flow(gauge, X, "wilson", n_steps=n, in_place=True), twin().flow(gauge, X, "wilson", n_steps=n))
