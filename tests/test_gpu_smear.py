"""GPU tier of gauge smearing: libquda_b200 against the host twin bit for bit in fp64 and fp32, for every kind and ignored
direction on the CPU tier's shapes and on 16^3x32; stout against the gauge force plus the link update, SU(3) output, the
ignored direction and time slices, gauge covariance and the boundary sign again through quda_b200.gauge.smear on device
tensors; the measurement rows of smear(meas_interval=...); and a clover CG solve on stout-smeared HMC links."""
import numpy as np
import pytest
import torch

import flow_ref as FR
import gauge_cases as GC
import smear_cases as SC
from quda_b200 import dirac as DR
from quda_b200 import gauge as GP
from quda_b200 import lib as L

pytestmark = pytest.mark.gpu


def lib():
    return SC.Runner(L.load(), "b200", dev=True)


twin = SC.twin


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("X", SC.SHAPES)
@pytest.mark.parametrize("kind", SC.KINDS)
@pytest.mark.parametrize("field", sorted(SC.FIELDS))
def test_library_matches_twin(X, kind, field):
    gauge = SC.FIELDS[field](X, 31)
    for ign in SC.IGNORE + [4]:
        for prec in (8, 4):
            got = lib().smear(gauge, X, kind, dir_ignore=ign, prec=prec)
            assert np.array_equal(got, twin().smear(gauge, X, kind, dir_ignore=ign, prec=prec)), (ign, prec)
            assert np.array_equal(got, lib().smear(gauge, X, kind, dir_ignore=ign, prec=prec))  # repeated calls
            assert np.array_equal(got, lib().smear(gauge, X, kind, dir_ignore=ign, prec=prec, in_place=True))


@pytest.mark.parametrize("kind", SC.KINDS)
def test_library_matches_twin_16x16x16x32(kind):
    X = (16, 16, 16, 32)
    gauge = GC.haar_links(X, 5)
    for ign in (-1, 3):
        for prec in (8, 4):
            got = lib().smear(gauge, X, kind, n_steps=1, dir_ignore=ign, prec=prec)
            assert np.array_equal(got, twin().smear(gauge, X, kind, n_steps=1, dir_ignore=ign, prec=prec)), (ign, prec)


# ------------------------------------------------------------------ the checks through quda_b200.gauge
def test_stout_is_force_plus_update_through_python():
    X = (4, 6, 8, 10)
    g = dev(GC.haar_links(X, 5))
    V = int(np.prod(X))
    mom = torch.zeros((V, 4, 10), dtype=torch.float64, device="cuda")
    paths, coeffs = GP.FLOW_ACTIONS["wilson"]
    GP.gauge_force(mom, g, paths, coeffs, 0.1, X=X)
    want = GP.update_gauge_field(g, mom, 1.0, X=X)
    got, rows = GP.smear(g, "stout", 1, X=X, rho=0.1, dir_ignore=4)
    assert torch.equal(got, want) and rows == []


@pytest.mark.parametrize("kind", SC.KINDS)
def test_checks_through_python(kind):
    X = (4, 6, 8, 10)
    gauge = GC.haar_links(X, 8)
    c = SC.COEFFS[kind]
    ign = GP.SMEAR_KINDS[kind][2]  # performGaugeSmearQuda's default
    f = GP.smear(dev(gauge), kind, SC.STEPS, X=X, **c)[0].cpu().numpy()
    assert np.array_equal(f, twin().smear(gauge, X, kind, dir_ignore=ign))
    assert max(SC.su3_deviation(f)) <= 1e-13
    # t ignored: the t links are copied, and one time slice changes nothing outside it
    ft = GP.smear(dev(gauge), kind, SC.STEPS, X=X, dir_ignore=3, **c)[0].cpu().numpy()
    assert np.array_equal(ft[3], gauge[3])
    other = np.array(gauge)
    sl = SC.time_slice_sites(X, 2)
    other[:, sl] = GC.haar_links(X, 9)[:, sl]
    fo = GP.smear(dev(other), kind, SC.STEPS, X=X, dir_ignore=3, **c)[0].cpu().numpy()
    rest = np.setdiff1d(np.arange(int(np.prod(X))), sl)
    assert np.array_equal(ft[:, rest], fo[:, rest])
    # gauge covariance, the plaquette, the boundary sign, in place
    gt = FR.random_su3((X[3], X[2], X[1], X[0]), 9)
    g2 = dev(FR.gauge_transform(gauge, X, gt))
    f2 = GP.smear(g2, kind, SC.STEPS, X=X, **c)[0]
    assert np.abs(f2.cpu().numpy() - FR.gauge_transform(f, X, gt)).max() <= 1e-12
    assert np.allclose(GP.plaquette(f2, X=X), GP.plaquette(dev(f), X=X), rtol=1e-12, atol=0)
    ga = dev(GC.antiperiodic(gauge, X))
    fa, _ = GP.smear(ga, kind, SC.STEPS, X=X, **c)
    assert np.array_equal(fa.cpu().numpy(), GC.antiperiodic(f, X))
    same, _ = GP.smear(ga, kind, SC.STEPS, X=X, out=ga, **c)
    assert same is ga and torch.equal(ga, fa)


def test_measurement_rows():
    X = (4, 6, 8, 10)
    g = dev(GC.haar_links(X, 3))
    out, rows = GP.smear(g, "ovrimp_stout", 6, X=X, meas_interval=2, **SC.COEFFS["ovrimp_stout"])
    assert [r[0] for r in rows] == [0, 2, 4, 6]
    u = g
    for k, (step, plaq, energy, q) in enumerate(rows):
        if k:
            u = GP.gauge_smear(torch.empty_like(g), u, "ovrimp_stout", 2, X=X, **SC.COEFFS["ovrimp_stout"])
        o = GP.gauge_observables(u, X=X)
        assert (plaq, energy, q) == (o["plaquette"], o["energy"], o["qcharge"])
    assert torch.equal(out, u)
    assert all(b[1][0] > a[1][0] for a, b in zip(rows, rows[1:]))  # smearing raises the plaquette
    with pytest.raises(L.B200Error):
        GP.smear(g, "wilson", 1, X=X)


# ------------------------------------------------------------------ smeared-link fermions
def test_clover_solve_on_stout_smeared_hmc_links():
    from test_gpu_gauge import X8, Hmc
    hmc = Hmc()
    U, _ = hmc.leapfrog(hmc.U0, hmc.mom0, 10)
    smeared, rows = GP.smear(U, "stout", 5, X=X8, rho=0.1, dir_ignore=4, meas_interval=5)
    print("plaquette before / after 5 stout steps:", rows[0][1][0], rows[1][1][0])
    assert rows[1][1][0] > rows[0][1][0]
    for links in (U, smeared):
        op, _ = hmc.operator(links)
        x = hmc.P.empty(1)
        p = DR.invert_cg(op, None, x, hmc.phi, tol=1e-10)
        print(f"CG: {p.iter} iterations, true residual {p.true_res:.3e}")
        assert p.true_res <= 1e-9 and p.iter < 10000
