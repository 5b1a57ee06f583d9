"""CPU tier of the per-element error bounds (tests/precise.py): the reference against the pinned oracle, the decoders
against the marshaling, the checker against deliberately wrong outputs, and the host twin of the site code under the
bound for every precision x reconstruction x operator on adversarial fields."""
import numpy as np
import pytest

import oracle
import precise as PR
import precise_cases as PC
from common import HostMem, PREC_NAME, twin_backend
from quda_b200 import fields as F

SHAPES = [(8, 8, 8, 8), (6, 10, 4, 14), (2, 4, 2, 6)]


def _dr(v):
    return PR.to_degrand_rossi(v).astype(np.float64)


# ---------------------------------------------------------------------------------------------- the reference itself
@pytest.mark.parametrize("X", [(4, 6, 4, 8), (6, 10, 4, 14)])
def test_reference_agrees_with_oracle(X):
    """The oracle is pinned bit for bit to the reference's host code.  On fp64 inputs it must agree with the long-double
    reference within the fp64 bound of every operator, seen as one more fp64 implementation."""
    Fs = PC.Fields(X, 8, 18, HostMem, seed=7, anisotropy=1.3, clover="near")
    s, xs = PR.gaussian_spinor(X, 1), PR.gaussian_spinor(X, 2)
    _, psi = Fs.spinor(s)
    _, x = Fs.spinor(xs)
    kappa, mu = 0.12195, 0.1
    for parity in (0, 1):
        for dagger in (0, 1):
            got = PR.from_degrand_rossi(oracle.wil_dslash(Fs.gauge, s, X, parity, dagger), np.clongdouble)
            PR.assert_within(got, PR.wilson(Fs.G, psi, X, parity, dagger, 8), 8, f"oracle dslash p={parity} d={dagger}")
            got = PR.from_degrand_rossi(oracle.clover_dslash(Fs.gauge, oracle.clover_invert(Fs.clover), s, X, parity,
                                                             dagger), np.clongdouble)
            PR.assert_within(got, PR.clover_pc(Fs.G, Fs.A, psi, X, parity, dagger, 8, True), 8, "oracle clover-pc")
            tm = oracle.twist_gamma5(xs, kappa, mu, dagger) - kappa * oracle.wil_dslash(Fs.gauge, s, X, parity, dagger)
            got = PR.from_degrand_rossi(tm, np.clongdouble)
            PR.assert_within(got, PR.twisted_mass(Fs.G, psi, X, parity, dagger, 8, -kappa, 2 * kappa * mu, x), 8,
                             "oracle twisted mass")
        got = PR.from_degrand_rossi(oracle.apply_clover(Fs.clover, s, X, parity), np.clongdouble)
        PR.assert_within(got, PR.clover_apply(Fs.A, psi, parity, False, True, 8), 8, "oracle A x")
        got = PR.from_degrand_rossi(oracle.apply_clover(oracle.clover_invert(Fs.clover), s, X, parity), np.clongdouble)
        PR.assert_within(got, PR.clover_apply(Fs.A, psi, parity, True, True, 8), 8, "oracle A^-1 x")
    for dagger in (0, 1):
        for inverse in (False, True):
            got = PR.from_degrand_rossi(oracle.twist_gamma5(s, kappa, mu, dagger, inverse), np.clongdouble)
            res = PR.twist(psi, *PR.twist_coefficients(kappa, mu, dagger, inverse), 8)
            # The oracle derives its own twist coefficients from kappa and mu and rotates in the DeGrand-Rossi basis;
            # it agrees to a few 1e-15 of the output, above the 3-rounding bound of the kernels' site-local twist, so
            # the twist is pinned here by relative agreement.
            assert np.abs(got - res.ref).max() <= 1e-14 * np.abs(res.ref).max(), "oracle twist"
    full = PR.gaussian_spinor(X, 3, nparity=2)
    M = oracle.wil_mat(Fs.gauge, full, X, kappa, 0)
    for parity in (0, 1):
        _, pin = Fs.spinor(full[(1 - parity) * Fs.Vh:(2 - parity) * Fs.Vh])
        _, pout = Fs.spinor(full[parity * Fs.Vh:(parity + 1) * Fs.Vh])
        got = PR.from_degrand_rossi(M[parity * Fs.Vh:(parity + 1) * Fs.Vh], np.clongdouble)
        PR.assert_within(got, PR.wilson(Fs.G, pin, X, parity, 0, 8, -kappa, pout), 8, "oracle full-field M")


def test_hermitian_inverse_and_condition():
    c = PR.hpd_clover((2, 2, 2, 2), 3, 1e3)
    blocks = np.zeros((16, 2, 6, 6), np.clongdouble)
    for i in range(6):
        blocks[..., i, i] = c[..., i]
    for i, j, k in PR.TRI:
        blocks[..., i, j] = c[..., k] + 1j * c[..., k + 1]
        blocks[..., j, i] = c[..., k] - 1j * c[..., k + 1]
    inv = PR.hermitian_inverse(blocks)
    eye = np.broadcast_to(np.eye(6), blocks.shape)
    assert np.abs(blocks @ inv - eye).max() < 1e-15
    assert np.allclose(PR.condition(blocks), 1e3, rtol=1e-9)


# ---------------------------------------------------------------------------------------------- decoders
@pytest.mark.parametrize("prec", [8, 4, 2])
def test_decoders_invert_the_marshaling(prec):
    X = (6, 10, 4, 14)
    Vh = F.volume_cb(X)
    s = PR.gaussian_spinor(X, 4, spread=30)
    native = F.rotate_basis(s, True).reshape(Vh, 12, 2)
    v, norm = PR.decode_spinor(F.spinor_to_native(s, prec), Vh, prec)
    want = native[..., 0] + 1j * native[..., 1]
    if prec == 2:
        d = np.abs(v.reshape(Vh, 12) - want)
        # half an LSB per component (re and im separately, sqrt 2 in modulus), plus the fp32 roundings of the value,
        # the scale 32767 / mx, the scaled value and the norm: 4 u relative, times |q| <= 32767 LSB
        assert np.all(d <= (0.5 + 4 * 2.0 ** -24 * 32767) * np.sqrt(2) * norm[:, None])
    else:
        cast = want.real.astype(F.real_dtype(prec)) + 1j * want.imag.astype(F.real_dtype(prec))
        assert np.array_equal(v.reshape(Vh, 12), cast.astype(v.dtype))
    g = PR.random_gauge(X, 5, anisotropy=2.38, antiperiodic_t=True)
    buf, meta = F.gauge_to_native(g, X, prec, 18)
    G = PR.decode_gauge(buf, X, prec, 18, meta, 2.38, -1)
    host = (g[..., 0] + 1j * g[..., 1]).reshape(4, 2, Vh, 3, 3).transpose(1, 0, 2, 3, 4)
    if prec == 2:
        assert np.abs(G.U[:, :, :Vh] - host).max() <= 0.5 * np.sqrt(2) * meta["link_max"] / 32767 * (1 + 1e-6)
    else:
        cast = host.real.astype(F.real_dtype(prec)) + 1j * host.imag.astype(F.real_dtype(prec))
        assert np.array_equal(G.U[:, :, :Vh], cast.astype(G.U.dtype))
    for recon in (12, 8):
        if prec == 2:
            continue
        Gr = PR.decode_gauge(*F.gauge_to_native(g, X, prec, recon)[:1], X, prec, recon, meta, 2.38, -1)
        assert np.abs(Gr.U[:, :, :Vh] - host).max() < (1e-12 if prec == 8 else 1e-5), f"recon-{recon} reconstruction"


# ---------------------------------------------------------------------------------------------- the checker
def _twin_half_case():
    be = twin_backend()
    Fs = PC.Fields((6, 10, 4, 14), 2, 12, HostMem, seed=11)
    din, psi = Fs.spinor(PR.gaussian_spinor(Fs.X, 12))
    out = PC.apply_op(Fs, "wilson", be, 0, 0, din)
    got, norm = Fs.read(out, with_norm=True)
    return Fs, got, norm, PR.wilson(Fs.G, psi, Fs.X, 0, 0, 2)


def _old_metric_accepts(res, got, prec, recon):
    _, dev, _ = oracle.compare_spinor(_dr(res.ref), _dr(got))
    return dev <= oracle.tolerance(PREC_NAME[prec], recon)


def test_checker_catches_what_the_old_metric_accepts():
    Fs, got, norm, res = _twin_half_case()
    assert PR.ratio(got, res, 2) <= 1
    scaled = got * (32767 / 32768)
    assert PR.ratio(scaled, res, 2) > 1, "a 3e-5 mis-scale of half precision must be caught"
    assert _old_metric_accepts(res, scaled, 2, 12), "documents the gap: compareSpinor accepts a 3e-5 mis-scale"
    site = int(np.argmax(norm))
    moved = got.copy()
    moved[site, 2, 1] += 2 * norm[site]
    assert PR.ratio(moved, res, 2) > 1, "a 2-LSB error in one element must be caught"
    assert _old_metric_accepts(res, moved, 2, 12), "documents the gap: compareSpinor accepts a 2-LSB error"
    small = int(np.argmin(norm))
    moved = got.copy()
    moved[small, 0, 0] += 2 * norm[small]
    assert PR.ratio(moved, res, 2) > 1, "a 2-LSB error at the smallest site must be caught"

    be = twin_backend()
    F8 = PC.Fields((6, 10, 4, 14), 8, 18, HostMem, seed=11)
    din, psi = F8.spinor(PR.gaussian_spinor(F8.X, 12))
    got8 = F8.read(PC.apply_op(F8, "wilson", be, 1, 1, din))
    res8 = PR.wilson(F8.G, psi, F8.X, 1, 1, 8)
    assert PR.ratio(got8, res8, 8) <= 1
    assert PR.ratio(got8 * (1 + 1e-13), res8, 8) > 1, "a 1e-13 relative error in fp64 must be caught"


def test_checker_catches_a_dropped_u0_on_the_last_time_slice():
    """recon-12 with anisotropy != 1 and antiperiodic t: an output computed as if the last time slice had no u0 factor
    (row 2 not negated there) must fail, while the twin's output passes"""
    be = twin_backend()
    X = (4, 6, 4, 8)
    Fs = PC.Fields(X, 4, 12, HostMem, seed=13, anisotropy=1.7, antiperiodic_t=True)
    din, psi = Fs.spinor(PR.gaussian_spinor(X, 14))
    res = PR.wilson(Fs.G, psi, X, 0, 0, 4)
    assert PR.ratio(Fs.read(PC.apply_op(Fs, "wilson", be, 0, 0, din)), res, 4) <= 1
    gbuf, gmeta = F.gauge_to_native(Fs.gauge, X, 4, 12)
    wrong = PR.decode_gauge(gbuf, X, 4, 12, gmeta, 1.7, -1, last_ts=False)
    bad = PR.wilson(wrong, psi, X, 0, 0, 4).ref
    assert PR.ratio(bad, res, 4) > 1


# ---------------------------------------------------------------------------------------------- host twin under the bound
GAUGES = {"haar": dict(), "eps1e-2": dict(eps=1e-2), "eps1e-4": dict(eps=1e-4),
          "aniso": dict(anisotropy=2.38, antiperiodic_t=False)}


@pytest.mark.parametrize("prec", [8, 4, 2])
@pytest.mark.parametrize("recon", [18, 12, 8])
@pytest.mark.parametrize("gauge", list(GAUGES))
def test_twin_wilson_under_bound(prec, recon, gauge):
    be = twin_backend()
    for i, X in enumerate(SHAPES):
        Fs = PC.Fields(X, prec, recon, HostMem, seed=20 + i, **GAUGES[gauge])
        for kind in ("gauss", "spread", "points"):
            parity, dagger = i % 2, (i + len(kind)) % 2
            PC.check_op(Fs, "wilson", be, parity, dagger, kind=kind, xpay=(kind == "spread"),
                        what=f"wilson X={X} {kind} p={parity} d={dagger}")


def test_twin_half_recon18_link_max_above_one():
    """spatial links are divided by the anisotropy: 1/2.38 makes them exceed 1, so half recon-18 needs link_max > 1"""
    be = twin_backend()
    Fs = PC.Fields((6, 10, 4, 14), 2, 18, HostMem, seed=3, anisotropy=1 / 2.38, antiperiodic_t=False)
    assert Fs.U.meta["link_max"] > 1
    for parity in (0, 1):
        PC.check_op(Fs, "wilson", be, parity, 1 - parity, kind="spread", xpay=True)


CLOVERS = {"near-compressed": dict(clover="near", compressed=True, dynamic=True),
           "hpd10-dynamic": dict(clover=10.0, compressed=False, dynamic=True),
           "hpd1e3-dynamic": dict(clover=1e3, compressed=False, dynamic=True),
           "hpd1e3-static": dict(clover=1e3, compressed=False, dynamic=False)}


@pytest.mark.parametrize("prec", [8, 4, 2])
@pytest.mark.parametrize("recon", [18, 12, 8])
@pytest.mark.parametrize("clover", list(CLOVERS))
def test_twin_clover_under_bound(prec, recon, clover):
    be = twin_backend()
    X = SHAPES[(prec + recon) % 3]
    Fs = PC.Fields(X, prec, recon, HostMem, seed=40, **CLOVERS[clover])
    PC.check_op(Fs, "clover", be, 0, 1, kind="spread")
    PC.check_op(Fs, "clover_pc", be, 1, 0, kind="gauss")
    PC.check_op(Fs, "clover_pc", be, 0, 0, kind="points", xpay=True)
    for inverse in (False, True):
        PC.check_clover_apply(Fs, be, inverse, kind="spread")


@pytest.mark.parametrize("prec", [8, 4, 2])
@pytest.mark.parametrize("recon", [18, 12, 8])
@pytest.mark.parametrize("mu", [0.1, 2.0])
def test_twin_twisted_mass_under_bound(prec, recon, mu):
    be = twin_backend()
    X = SHAPES[(prec + recon + int(mu)) % 3]
    Fs = PC.Fields(X, prec, recon, HostMem, seed=60)
    for dagger in (0, 1):
        PC.check_op(Fs, "tm", be, dagger, dagger, kind="spread", mu=mu)
        for inverse in (False, True):
            PC.check_twist_gamma(Fs, be, dagger, inverse, mu=mu, kind="spread")


@pytest.mark.parametrize("prec,recon", [(8, 18), (4, 12), (2, 8), (2, 18)])
@pytest.mark.parametrize("comm_dim", [(1, 0, 0, 0), (0, 0, 0, 1), (1, 1, 1, 1)])
@pytest.mark.parametrize("split", [None, "sites", "reference"])
def test_twin_partitioned_under_bound(prec, recon, comm_dim, split):
    PC.check_partitioned(PC.Fields((4, 6, 4, 8), prec, recon, HostMem, seed=70), "wilson", twin_backend(), comm_dim, split)


def test_twin_partitioned_clover_pc_under_bound():
    Fs = PC.Fields((4, 6, 4, 8), 2, 12, HostMem, seed=71, clover="near")
    PC.check_partitioned(Fs, "clover_pc", twin_backend(), (1, 1, 1, 1), "tiles", dagger=0)


@pytest.mark.parametrize("prec,recon", [(8, 18), (4, 12), (2, 8)])
@pytest.mark.parametrize("flavour", ["thread", "cta"])
def test_twin_multi_rhs_under_bound(monkeypatch, prec, recon, flavour):
    monkeypatch.setenv("B200_MRHS_MODE", flavour)
    PC.check_multi(PC.Fields((8, 4, 6, 4), prec, recon, HostMem, seed=80), "wilson", twin_backend(), 5)


# ---------------------------------------------------------------------------------------------- zeros stay zeros
@pytest.mark.parametrize("prec", [8, 4, 2])
def test_unreached_sites_are_exact_zeros(prec):
    be = twin_backend()
    X = (8, 8, 8, 8)
    Fs = PC.Fields(X, prec, 12, HostMem, seed=90)
    din, psi = Fs.spinor(PC.spinor_kind(X, "points", 91, prec))
    got, norm = Fs.read(PC.apply_op(Fs, "wilson", be, 1, 0, din), with_norm=True)
    res = PR.wilson(Fs.G, psi, X, 1, 0, prec)
    dead = np.all(res.bound == 0, axis=(1, 2))
    assert dead.sum() > Fs.Vh // 2
    assert np.all(got[dead] == 0)
    if prec == 2:
        assert np.all(norm[dead] == 0) and np.all(np.isfinite(got))
    PR.assert_within(got, res, prec, "point sources")
