"""GPU tier of the per-element error bounds (tests/precise.py): every kernel family of libquda_b200.so against the
high-precision reference on adversarial fields, plus two edge tests of the half-precision format that only the GPU
path can exercise (the PRMT / magic-add int16 decode and the __fdividef block-float store)."""
import numpy as np
import pytest

import precise as PR
import precise_cases as PC
from common import CudaMem
from quda_b200 import dslash as D
from quda_b200 import fields as F
from quda_b200 import lib as L

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _native_loaded():
    import torch
    assert torch.cuda.is_available(), "GPU tier needs a CUDA device"
    lib = L.load()
    before = lib.b200_launch_count()
    yield
    assert lib.b200_launch_count() > before, "no kernel from libquda_b200.so was launched"


GAUGES = {"haar": dict(), "eps1e-4": dict(eps=1e-4), "aniso": dict(anisotropy=2.38, antiperiodic_t=False)}


@pytest.mark.parametrize("prec", [8, 4, 2])
@pytest.mark.parametrize("recon", [18, 12, 8])
@pytest.mark.parametrize("gauge", list(GAUGES))
def test_interior_kernel(prec, recon, gauge):
    for i, X in enumerate([(8, 8, 8, 8), (6, 10, 4, 14)]):
        Fs = PC.Fields(X, prec, recon, CudaMem, seed=120 + i, **GAUGES[gauge])
        for kind in ("gauss", "spread", "points"):
            PC.check_op(Fs, "wilson", None, i, len(kind) % 2, kind=kind, xpay=(kind == "gauss"))


def test_half_recon18_link_max_above_one():
    Fs = PC.Fields((8, 8, 8, 8), 2, 18, CudaMem, seed=3, anisotropy=1 / 2.38, antiperiodic_t=False)
    assert Fs.U.meta["link_max"] > 1
    PC.check_op(Fs, "wilson", None, 1, 0, kind="spread", xpay=True)


@pytest.mark.parametrize("prec,recon", [(8, 18), (4, 12), (2, 8), (2, 12)])
@pytest.mark.parametrize("comm_dim", [(1, 0, 0, 0), (0, 0, 0, 1), (1, 1, 1, 1)])
@pytest.mark.parametrize("split", [None, "sites", "tiles", "reference"])
def test_partitioned(prec, recon, comm_dim, split):
    Fs = PC.Fields((4, 6, 4, 8), prec, recon, CudaMem, seed=130)
    PC.check_partitioned(Fs, "wilson", None, comm_dim, split)


def test_partitioned_clover_pc():
    Fs = PC.Fields((4, 6, 4, 8), 2, 12, CudaMem, seed=131, clover="near")
    PC.check_partitioned(Fs, "clover_pc", None, (1, 1, 1, 1), "tiles", dagger=0)


@pytest.mark.parametrize("flavour", ["thread", "cta"])
def test_multi_rhs(monkeypatch, flavour):
    monkeypatch.setenv("B200_MRHS_MODE", flavour)
    for prec, recon in ((4, 12), (2, 8)):
        PC.check_multi(PC.Fields((16, 4, 4, 4), prec, recon, CudaMem, seed=140), "wilson", None, 7)


@pytest.mark.parametrize("prec,recon", [(4, 12), (8, 18)])
def test_tma_kernel(monkeypatch, prec, recon):
    monkeypatch.setenv("B200_TMA", "2")  # fail rather than fall back to the gather kernel
    Fs = PC.Fields((16, 8, 4, 6), prec, recon, CudaMem, seed=150, eps=1e-2)
    for kind in ("gauss", "spread", "points"):
        PC.check_op(Fs, "wilson", None, 0, 1, kind=kind)


CLOVERS = {"near-compressed-dynamic": dict(clover="near", compressed=True, dynamic=True),
           "hpd1e3-dynamic": dict(clover=1e3, compressed=False, dynamic=True),
           "near-compressed-static": dict(clover="near", compressed=True, dynamic=False),
           "hpd1e3-static": dict(clover=1e3, compressed=False, dynamic=False)}


@pytest.mark.parametrize("prec", [8, 4, 2])
@pytest.mark.parametrize("clover", list(CLOVERS))
def test_clover(prec, clover):
    Fs = PC.Fields((8, 4, 6, 4), prec, 12, CudaMem, seed=160, **CLOVERS[clover])
    for inverse in (False, True):
        PC.check_clover_apply(Fs, None, inverse, kind="spread")
    PC.check_op(Fs, "clover", None, 0, 1, kind="spread")
    PC.check_op(Fs, "clover_pc", None, 1, 0, kind="gauss", xpay=True)


@pytest.mark.parametrize("prec", [8, 4, 2])
@pytest.mark.parametrize("mu", [0.1, 2.0])
def test_twist(prec, mu):
    Fs = PC.Fields((8, 4, 6, 4), prec, 12, CudaMem, seed=170)
    for dagger in (0, 1):
        PC.check_op(Fs, "tm", None, dagger, dagger, kind="spread", mu=mu)
        for inverse in (False, True):
            PC.check_twist_gamma(Fs, None, dagger, inverse, mu=mu, kind="spread")


def test_bench_workload_32_fp32_recon12():
    """the bench.py workload: 32^4, fp32, recon-12, against the float64 reference"""
    Fs = PC.Fields((32, 32, 32, 32), 4, 12, CudaMem, seed=137)
    PC.check_op(Fs, "wilson", None, 0, 0, kind="gauss")


def test_clover_pc_16_half_recon8():
    Fs = PC.Fields((16, 16, 16, 16), 2, 8, CudaMem, seed=138, clover="near")
    PC.check_op(Fs, "clover_pc", None, 1, 0, kind="gauss")


def _payload_spinor(X):
    """half spinor buffer whose int16 planes hold every value of [-32768, 32767] at every lane position of the
    16-byte vector, over the sites; power-of-two norms"""
    Vh = F.volume_cb(X)
    assert Vh >= 65536
    site = np.arange(Vh)
    q = np.empty((3, Vh, 8), np.int16)
    for p in range(3):
        for lane in range(8):
            q[p, :, lane] = ((site + 9973 * (8 * p + lane)) % 65536 - 32768).astype(np.int16)
    norm = np.exp2(site % 24 - 12).astype(np.float32)
    return np.concatenate([q.view(np.uint8).ravel(), norm.view(np.uint8).ravel()]), q, norm


def test_every_int16_payload_decodes_exactly():
    import torch
    X = (16, 16, 16, 32)
    Vh = F.volume_cb(X)
    buf, q, norm = _payload_spinor(X)
    field = D.ColorSpinorField(CudaMem.put(buf), X, 2, 1)
    host = torch.zeros((Vh, 4, 3, 2), dtype=torch.float64, device="cuda")
    D.copy_spinor(field, host, False)
    torch.cuda.synchronize()
    # undo the DeGrand-Rossi rotation in long double: the native value must be q * norm to far better than 1 LSB
    back = PR.from_degrand_rossi(host.cpu().numpy(), np.clongdouble).reshape(Vh, 12)
    flat = np.stack([back.real, back.imag], -1).reshape(Vh, 24)
    want = q.transpose(1, 0, 2).reshape(Vh, 24).astype(np.longdouble)
    t = flat / norm.astype(np.longdouble)[:, None]
    assert np.abs(t - want).max() < 1e-6, "an int16 payload decoded to the wrong value"
    assert np.array_equal(np.rint(t).astype(np.int64), want.astype(np.int64))
    Fs = PC.Fields(X, 2, 12, CudaMem, seed=180)
    psi = PR.decode_spinor(buf, Vh, 2)[0]
    out = Fs.empty()
    D.ApplyWilson(out, field, Fs.U, 0.0, None, 1, 0)
    PR.assert_within(Fs.read(out), PR.wilson(Fs.G, psi, X, 1, 0, 2), 2, "Wilson on every int16 payload")


def test_tiny_sites_stay_finite():
    """site maxima below ~1e-34 overflow 32767 / mx in __fdividef: a documented limit of the block-float format.  The
    stored values must still decode to finite numbers no larger than the site maximum."""
    X = (8, 4, 4, 4)
    Vh = F.volume_cb(X)
    s = PR.gaussian_spinor(X, 190)
    s *= np.exp2(-120.0 - (np.arange(Vh) % 6)).reshape(Vh, 1, 1, 1)
    Fs = PC.Fields(X, 2, 18, CudaMem, seed=191)
    din, psi = Fs.spinor(s)
    out = Fs.empty()
    D.ApplyTwistGamma(out, din, 0.12195, 0.1, 0, False)
    got = Fs.read(out)
    mx = np.max(np.abs(PR.twist(psi, *PR.twist_coefficients(0.12195, 0.1, 0, False), 2).ref), axis=(1, 2))
    assert np.all(np.isfinite(got))
    assert np.all(np.abs(got).max(axis=(1, 2)) <= mx * (1 + 1e-6))
