"""GPU tier (-m gpu): libquda_b200.so through its C ABI against the CPU oracle on identical seeded fields,
using the reference's comparison metric and tolerances (fp64 1e-11 -- we also assert the north star's 1e-12 --,
fp32 1e-4, half 1e-3, x10 for recon-8 half)."""
import os

import numpy as np
import pytest

import ops
import oracle
from common import CudaMem, Problem, assert_close
from quda_b200 import dslash as D
from quda_b200 import lib as L

pytestmark = pytest.mark.gpu

PRECS = [8, 4, 2]
RECONS = [18, 12, 8]


@pytest.fixture(scope="module", autouse=True)
def _native_loaded():
    import torch
    assert torch.cuda.is_available(), "GPU tier needs a CUDA device"
    lib = L.load()
    before = lib.b200_launch_count()
    yield
    assert lib.b200_launch_count() > before, "no kernel from libquda_b200.so was launched"


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("recon", RECONS)
@pytest.mark.parametrize("X", [(8, 8, 8, 8), (4, 6, 8, 10)])
def test_wilson_dslash_vs_oracle(prec, recon, X):
    dev = ops.check_wilson_dslash(CudaMem, None, prec, recon, X)
    if prec == 8:
        assert dev <= 1e-12


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("recon", [18, 12, 8])
def test_wilson_xpay_and_tiles(prec, recon):
    """out = x + a D in, for several launch tilings including ragged ones (tile does not divide the lattice)."""
    X = (8, 6, 4, 6)
    P = Problem(X, prec, recon, CudaMem, anisotropy=1.7, antiperiodic_t=True)
    kappa = 0.12195
    s, xs = P.spinor(seed=3), P.spinor(seed=4)
    ref = ops.reference(P, "wilson", s, 1, 0, xs, -kappa)
    for tile in (None, (4, 1, 1, 1), (4, 6, 1, 1), (2, 2, 2, 2), (3, 4, 4, 4), (4, 6, 4, 3)):
        out = P.empty()
        D.ApplyWilson(out, P.to_dev(s), P.U, -kappa, P.to_dev(xs), 1, 0, tile=tile)
        assert_close(ref, P.to_host(out), prec, recon, f"xpay tile={tile}")


@pytest.mark.parametrize("prec", PRECS)
def test_wilson_full_field(prec):
    """nParity = 2: both parities in one call (DiracWilson::M path, lib/dirac_wilson.cpp:44-61)."""
    X = (8, 4, 4, 6)
    P = Problem(X, prec, 12, CudaMem)
    kappa = 0.11
    full = P.spinor(seed=9, nparity=2)
    out = P.empty(2)
    inp = P.to_dev(full, 2)
    D.ApplyWilson(out, inp, P.U, -kappa, inp, D.QUDA_INVALID_PARITY, 0)
    ref = oracle.wil_mat(P.gauge, full, X, kappa, 0)
    assert_close(ref, P.to_host(out), prec, 12, "full-field M")


def test_argument_errors():
    X = (4, 4, 4, 4)
    P = Problem(X, 4, 12, CudaMem)
    s = P.to_dev(P.spinor())
    with pytest.raises(L.B200Error, match="alias"):
        D.ApplyWilson(s, s, P.U, 0.0, None, 0, 0)
    with pytest.raises(L.B200Error, match="x is null"):
        D.ApplyWilson(P.empty(), s, P.U, 0.5, None, 0, 0)
    with pytest.raises(L.B200Error, match="clover"):
        D.ApplyWilsonClover(P.empty(), s, P.U, D.CloverField(None, X, 4, dict(parity_stride_bytes=0, compressed=0,
                            diagonal=0.0, max_element=1.0)), 0.5, s, 0, 0)


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("host_dtype", ["float32", "float64"])
def test_device_side_spinor_marshaling(prec, host_dtype):
    """b200_copy_spinor (host interface order <-> native UKQCD order, on the device) against the numpy marshaling"""
    import torch
    from quda_b200 import fields as F
    X = (4, 6, 4, 8)
    P = Problem(X, prec, 12, CudaMem)
    s = P.spinor(seed=8).astype(host_dtype)
    dev_host_order = torch.from_numpy(s).cuda()
    nat = P.empty()
    D.copy_spinor(nat, dev_host_order, True)
    got = P.to_host(nat)                      # numpy: native -> host order
    assert_close(s, got, prec, 18, "to native")
    back = torch.zeros_like(dev_host_order)
    D.copy_spinor(P.to_dev(s), back, False)
    torch.cuda.synchronize()
    assert_close(s, back.cpu().numpy(), prec, 18, "from native")


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("recon", RECONS)
def test_device_side_gauge_marshaling(prec, recon):
    """b200_copy_gauge (QDP host order -> native packed order + ghost pad, on the device) against the numpy marshaling"""
    from quda_b200 import fields as F
    X = (4, 6, 4, 8)
    hp = 8 if prec == 8 else 4
    g = oracle.random_gauge(X, hp, seed=21, anisotropy=1.4)
    want, meta = F.gauge_to_native(g, X, prec, recon)
    U = D.load_gauge(g, X, prec, recon, anisotropy=1.4, t_boundary=-1)
    got = U.buf.cpu().numpy()
    assert U.meta["stride"] == meta["stride"] and U.meta["parity_stride_bytes"] == meta["parity_stride_bytes"]
    if prec == 2:
        d = np.abs(got.view(np.int16).astype(int) - want.view(np.int16).astype(int))
        assert d.max() <= 1
    else:
        a, b = got.view(F.real_dtype(prec)), want.view(F.real_dtype(prec))
        assert np.allclose(a, b, rtol=0, atol=1e-14 if prec == 8 else 2e-7)
    # and the loaded field drives the operator
    P = Problem(X, prec, recon, CudaMem, seed=21, anisotropy=1.4)
    s = P.spinor(seed=2)
    out = P.empty()
    D.ApplyWilson(out, P.to_dev(s), U, 0.0, None, 0, 0)
    assert_close(oracle.wil_dslash(P.gauge, s, X, 0, 0), P.to_host(out), prec, recon, "dslash on device-marshaled gauge")


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("compressed", [True, False])
def test_device_side_clover_marshaling(prec, compressed):
    from quda_b200 import fields as F
    X = (4, 4, 6, 4)
    hp = 8 if prec == 8 else 4
    c = oracle.random_clover(X, hp, seed=33)
    want, meta = F.clover_to_native(c, X, prec, compressed=compressed)
    A = D.load_clover(c, X, prec, compressed=compressed)
    got = A.buf.cpu().numpy()
    assert A.meta["parity_stride_bytes"] == meta["parity_stride_bytes"]
    assert abs(A.meta["diagonal"] - meta["diagonal"]) < 1e-6 and abs(A.meta["max_element"] - meta["max_element"]) < 1e-6 * meta["max_element"]
    if prec == 2:
        d = np.abs(got.view(np.int16).astype(int) - want.view(np.int16).astype(int))
        assert d.max() <= 1
    else:
        assert np.allclose(got.view(F.real_dtype(prec)), want.view(F.real_dtype(prec)), rtol=0, atol=1e-14 if prec == 8 else 2e-7)
    P = Problem(X, prec, 12, CudaMem, clover=True, compressed=compressed, dynamic=True)
    s = P.spinor(seed=2)
    out = P.empty()
    D.ApplyClover(out, P.to_dev(s), A, False, 1)
    assert_close(oracle.apply_clover(c, s.astype(c.dtype), X, 1), P.to_host(out), prec, 12, "A x on device-marshaled clover")
