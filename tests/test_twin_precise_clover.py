"""CPU tier of the per-element bounds of tests/precise_clover.py: the host twins of the clover build and the clover force
(the library's site code compiled for the CPU) on adversarial links, clover terms, spinors and lattice shapes, the
extended-lattice build for every border mask, and negative controls: deliberately wrong outputs, made by perturbing the
twins' results, that the checks must reject."""
import numpy as np
import pytest

import clover_build_ref as R
import clover_force_ref as CF
import precise as PR
import precise_clover as PCL
import precise_clover_cases as C


@pytest.fixture(scope="module")
def tier():
    return C.Tier(False)


@pytest.mark.parametrize("field", list(C.BUILD_FIELDS))
@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("shape", list(C.SHAPES))
def test_build(tier, shape, prec, field):
    C.check_build(tier, C.SHAPES[shape], prec, *C.BUILD_FIELDS[field])


@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("name", list(C.FORCE_CASES))
def test_force(tier, name, prec):
    C.check_force(tier, C.force_case(name, prec))


@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("shape", ["4x6x8x10", "6x2x4x6"])
def test_border(tier, shape, prec):
    C.check_border(tier, C.SHAPES[shape], prec)


def test_extend_periodic_matches_comm_layout():
    """the numpy halo has the extended lattice's QDP order: the link of every extended site is that of its wrapped
    interior site"""
    X, mask = (4, 6, 2, 4), (1, 0, 1, 1)
    g = np.arange(4 * int(np.prod(X)), dtype=np.float64).reshape(4, -1)
    ext, Xe = C.extend_periodic(g, X, mask)
    c = np.concatenate([C.F.cb_coords(Xe, p) for p in range(2)])
    w = [(c[:, d] - mask[d]) % X[d] for d in range(4)]
    lex = ((w[3] * X[2] + w[2]) * X[1] + w[1]) * X[0] + w[0]
    inv = np.empty(int(np.prod(X)), int)
    inv[C.comm._lex_of_sites(X)] = np.arange(int(np.prod(X)))
    assert np.array_equal(ext, g[:, inv[lex]])


# ---------------------------------------------------------------------------------------------- negative controls
def rejected(got, res, prec, what):
    r = PR.ratio(got, res, prec)
    print(f"{what}: max err/bound = {r:.3g} (must be > 1)")
    assert r > 1, f"{what}: a wrong output passed the check (max err/bound {r:.3g})"


def test_rejects_identity_on_smooth_links(tier):
    X = C.SHAPES["4x6x8x10"]
    gauge = C.gauge_field(X, "eps1e-5", 11, 4)
    A, _, _ = tier.build(gauge, X, 4, C.COEFF)
    res = PCL.clover_build(gauge, X, C.COEFF, 4)
    PR.assert_within(A, res, 4, "twin")
    one = np.zeros_like(A)
    one[..., :6] = 1
    rejected(one, res, 4, "A = 1 on eps = 1e-5 links")


@pytest.mark.parametrize("prec", [8, 4])
def test_rejects_wrong_leaf_orientation(tier, prec):
    """plane (2, 1) with its second leaf traversed backwards"""
    X = C.SHAPES["4x6x8x10"]
    gauge = C.gauge_field(X, "eps1e-2", 11, prec)

    def wrong(U, mu, nu):
        Q = PCL.leaf_sum(U, mu, nu)
        if (mu, nu) == (2, 1):
            s = lambda a, dm, dn: R.shift(R.shift(a, mu, dm), nu, dn)  # noqa: E731
            leaf = U[nu] @ R.dag(s(U[mu], -1, 1)) @ R.dag(s(U[nu], -1, 0)) @ s(U[mu], -1, 0)
            Q = Q - leaf + R.dag(leaf)
        return Q

    A, _, _ = tier.build(gauge, X, prec, C.COEFF)
    res = PCL.clover_build(gauge, X, C.COEFF, prec)
    G, TG = PCL.planes(gauge, X, prec, leaf=wrong)
    bad = PCL.build_from_planes(G, TG, X, C.COEFF, prec).ref
    rejected((A + (bad - res.ref)).astype(A.dtype), res, prec, "F21 from a reversed leaf")


@pytest.mark.parametrize("shape", ["4x6x8x10", "8^4"])
def test_rejects_trlog_summed_in_fp32(tier, shape):
    X = C.SHAPES[shape]
    A, _, tl = tier.build(C.gauge_field(X, "haar", 11, 8), X, 8, C.COEFF)
    Iv = PCL.Inverse(A, 8)
    res = Iv.trlog(X)
    PR.assert_within(np.array(tl), res, 8, "twin")
    d = np.real(np.diagonal(Iv.L, axis1=-2, axis2=-1)).astype(np.float64)
    logdet = (2 * np.log(d)).sum(-1).sum(-1)  # per site, double
    Vh = len(logdet) // 2
    got = np.array([np.cumsum(logdet[p * Vh:(p + 1) * Vh].astype(np.float32), dtype=np.float32)[-1] for p in range(2)])
    rejected(got.astype(np.float64), res, 8, "log det accumulated in fp32")


def _mom_delta(df, X):
    """the change of mom when the force changes by df [4][lex][3][3]"""
    fs = np.stack([R.from_lex(df[mu], X) for mu in range(4)], axis=1)
    return PCL.mom_sub_ta(np.zeros(fs.shape[:2] + (10,)), fs)


@pytest.mark.parametrize("prec", [8, 4])
def test_rejects_hop_force_along_the_wrong_direction(tier, prec):
    """the hopping force of U_y built from the neighbours along z"""
    case = C.ForceCase(C.SHAPES["4x6x8x10"], prec, 1, "gauss")
    got = tier.force(case, prec)
    ref = case.reference()
    PR.assert_within(got, ref.result, prec, "twin")
    xs, ps = [case.decoded(x) for x in case.xs], [case.decoded(p) for p in case.ps]
    U = PCL.links(case.gauge, case.X, prec)
    one, mu, nu = np.eye(4), 1, 2
    r = 0
    for x, p, c in zip(xs, ps, case.fc):
        r = r + c * (CF.outer(CF.spin(one + CF.GAMMA[mu], R.shift(x, nu, 1)), p)
                     + CF.outer(CF.spin(one - CF.GAMMA[mu], R.shift(p, nu, 1)), x))
    df = np.zeros_like(ref.f_hop)
    df[mu] = U[mu] @ r - ref.f_hop[mu]
    rejected(got + _mom_delta(df, case.X).astype(np.float64), ref.result, prec, "hop force of y from the z neighbour")


@pytest.mark.parametrize("prec", [8, 4])
def test_rejects_oprod_corner_at_x(tier, prec):
    """the insertion at the corner x + mu of the upper leaf reads oprod at x"""
    case = C.ForceCase(C.SHAPES["4x6x8x10"], prec, 3, "gauss")
    got = tier.force(case, prec)
    ref = case.reference()
    PR.assert_within(got, ref.result, prec, "twin")
    U = PCL.links(case.gauge, case.X, prec)
    df = []
    for mu in range(4):
        f = 0
        for nu in range(4):
            if nu == mu:
                continue
            Ot = ref.O[R.PLANES.index((max(mu, nu), min(mu, nu)))]
            s = lambda a, dm, dn: R.shift(R.shift(a, mu, dm), nu, dn)  # noqa: E731
            U1, U2, U3, U4 = U[mu], s(U[nu], 1, 0), s(U[mu], 0, 1), U[nu]
            f = f + (1.0 if nu > mu else -1.0) * (U1 @ (Ot - s(Ot, 1, 0)) @ U2 @ R.dag(U3) @ R.dag(U4))
        df.append(f)
    rejected(got + _mom_delta(np.stack(df), case.X).astype(np.float64), ref.result, prec, "oprod corner read at x")


@pytest.mark.parametrize("prec", [8, 4])
def test_rejects_a_few_hundred_ulp_at_the_smallest_sites(tier, prec):
    """300 ulp of the hopping force's update, on the 1% of links with the smallest force only"""
    case = C.ForceCase(C.SHAPES["6x2x4x6"], prec, 1, "spread")
    got = tier.force(case, prec, "hop")
    ref = case.reference("hop")
    PR.assert_within(got, ref.result, prec, "twin")
    b = ref.result.bound[..., 0]
    small = b <= np.quantile(b, 0.01)
    bad = got.copy()
    bad[small, :9] += 300 * PR.U_P[prec] * np.abs(got[small, :9]).max(-1, keepdims=True)
    rejected(bad, ref.result, prec, "300 ulp at the smallest sites")
