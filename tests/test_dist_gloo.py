"""CPU tier, world_size = 2 over gloo: process-grid topology, local slicing of global fields, face packing,
neighbour exchange and the interior + exterior split -- each rank computes its half of a global lattice with
the host twin and the gathered result must match the oracle on the GLOBAL lattice."""
import pytest

from dist_worker import run_ranks, worker


@pytest.fixture(scope="module", autouse=True)
def _twin_built():
    """build the host twin once in the parent: two freshly spawned ranks must not race to compile it"""
    from common import twin_backend
    twin_backend()


@pytest.mark.parametrize("grid_dims,Xl", [((1, 1, 1, 2), (4, 4, 4, 4)), ((2, 1, 1, 1), (4, 4, 6, 4)), ((1, 2, 1, 1), (4, 4, 4, 6))])
@pytest.mark.parametrize("prec,recon", [(8, 18), (4, 12), (2, 8)])
def test_two_rank_wilson_matches_global_oracle(grid_dims, Xl, prec, recon):
    res = run_ranks(worker, 2, (grid_dims, Xl, prec, recon), timeout=300)
    tol = {8: 1e-11, 4: 1e-4, 2: 1e-2}[prec]
    for r in res:
        assert r["dev"] <= tol, (r["rank"], r["dev"])


@pytest.mark.parametrize("grid_dims,Xl,prec,recon", [((1, 1, 1, 2), (4, 4, 4, 4), 8, 18), ((2, 1, 1, 1), (4, 4, 6, 4), 2, 12)])
def test_two_rank_batched_halo_matches_global_oracle(grid_dims, Xl, prec, recon):
    """a multi-RHS batch on a partitioned lattice: one batched exchange for 3 sources (HaloExchange(n_src=3))"""
    res = run_ranks(worker, 2, (grid_dims, Xl, prec, recon, "host", 2, 3), timeout=300)
    tol = {8: 1e-11, 4: 1e-4, 2: 1e-2}[prec]
    for r in res:
        assert r["dev"] <= tol, (r["rank"], r["dev"])


def test_process_grid_topology():
    from quda_b200.comm import ProcessGrid
    g = ProcessGrid((1, 2, 2, 2), 5)
    assert g.coords == [0, 1, 0, 1] and g.rank_of(g.coords) == 5
    assert g.neighbor(3, +1) == g.rank_of([0, 1, 0, 0]) and g.neighbor(1, -1) == g.rank_of([0, 0, 0, 1])
    assert ProcessGrid.default_dims(8) == [1, 2, 2, 2] and ProcessGrid.default_dims(2) == [1, 1, 1, 2]
    assert g.comm_dim() == [0, 1, 1, 1]
