"""CPU tier: the product's site code (compiled for the host, tests/hosttwin) against the oracle.
Same b200_dslash_args ABI, same native layouts, same argument validation as the CUDA library."""
import pytest

import ops
from common import HostMem, Problem, assert_close, twin_backend
from quda_b200 import dslash as D

PRECS = [8, 4, 2]
RECONS = [18, 12, 8]


@pytest.mark.parametrize("prec", PRECS)
@pytest.mark.parametrize("recon", RECONS)
@pytest.mark.parametrize("X", [(4, 4, 4, 4), (8, 4, 6, 2)])
def test_wilson_dslash(prec, recon, X):
    ops.check_wilson_dslash(HostMem, twin_backend(), prec, recon, X)


@pytest.mark.parametrize("tile", [(16, 2, 2, 1), (2, 2, 2, 2), (1, 4, 1, 2), (4, 1, 1, 1), (2, 8, 4, 2), (3, 4, 4, 2)])
def test_launch_tilings_cover_the_lattice(tile):
    """The host twin walks the same (grid, block) decomposition the CUDA launcher builds (launch.h::make_tile_map,
    dslash_site.h::tile_site): every tiling, including ragged ones and nt0 == 1, must visit each site exactly once."""
    be = twin_backend()
    X = (8, 6, 4, 6)
    P = Problem(X, 4, 12, HostMem)
    ops.wilson_vs_oracle(P, be, P.spinor(seed=2), 1, 0, f"tile {tile}", tile=tile)
    full = P.spinor(seed=3, nparity=2)
    out2 = P.empty(2)
    D.ApplyWilson(out2, P.to_dev(full, 2), P.U, 0.0, None, D.QUDA_INVALID_PARITY, 0, tile=tile, backend=be)
    assert_close(ops.full_dslash(P, full, 0), P.to_host(out2), 4, 12, f"full-field tile {tile}")


@pytest.mark.parametrize("X", [(2, 2, 2, 2), (2, 4, 2, 6), (4, 2, 2, 2), (16, 2, 4, 2)])
@pytest.mark.parametrize("prec,recon", [(8, 12), (4, 8), (2, 18)])
def test_degenerate_extents(X, prec, recon):
    """smallest legal lattices: extent 2 makes the forward and the backward neighbour the same site (and X0 = 2 leaves one
    checkerboard site per row); anisotropy + periodic t exercise the other u0 branch of the reconstruction"""
    be = twin_backend()
    P = Problem(X, prec, recon, HostMem, anisotropy=2.38, antiperiodic_t=False)
    for parity, dagger in ((0, 0), (1, 1)):
        s, xs = P.spinor(seed=7 + parity), P.spinor(seed=9)
        out = P.empty()
        D.ApplyWilson(out, P.to_dev(s), P.U, -0.1, P.to_dev(xs), parity, dagger, backend=be)
        assert_close(ops.reference(P, "wilson", s, parity, dagger, xs, -0.1), P.to_host(out), prec, recon, f"X={X} parity={parity}")
