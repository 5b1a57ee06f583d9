"""GPU tier: operator composition (DiracWilson[PC], DiracClover[PC]) and CG against the oracle's
wil_mat / wil_matpc / clover_mat / clover_matpc (the reference's --test Mat / MatPC / MatPCDagMatPC cases,
tests/dslash_test_utils.h:363-786) and a host-verified true residual as invert_test does
(tests/invert_test_gtest.hpp:107-128)."""
import pytest

import oracle
from common import CudaMem, Problem, assert_close
from quda_b200 import dirac as DR
from solvers import KAPPA, MU, X8, busy_default_stream, solve

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("prec", [8, 4])
def test_wilson_mat_and_matpc(prec):
    X = (4, 6, 4, 8)
    P = Problem(X, prec, 12, CudaMem)
    full = P.spinor(seed=3, nparity=2)
    op = DR.Dirac("wilson", P.U, KAPPA)
    for dagger in (0, 1):
        out = P.empty(2)
        op.M(out, P.to_dev(full, 2), dagger=dagger)
        assert_close(oracle.wil_mat(P.gauge, full, X, KAPPA, dagger), P.to_host(out), prec, 12, "wilson M")
    s = P.spinor(seed=4)
    for matpc in (DR.MATPC_EVEN_EVEN, DR.MATPC_ODD_ODD):
        pc = DR.Dirac("wilsonpc", P.U, KAPPA, matpc_type=matpc)
        for dagger in (0, 1):
            out = P.empty()
            pc.M(out, P.to_dev(s), dagger=dagger)
            assert_close(oracle.wil_matpc(P.gauge, s, X, KAPPA, matpc, dagger), P.to_host(out), prec, 12, "wilson Mpc")
        out = P.empty()
        pc.MdagM(out, P.to_dev(s))
        ref = oracle.wil_matpc(P.gauge, oracle.wil_matpc(P.gauge, s, X, KAPPA, matpc, 0), X, KAPPA, matpc, 1)
        assert_close(ref, P.to_host(out), prec, 12, "wilson MpcdagMpc")


@pytest.mark.parametrize("prec", [8, 4])
@pytest.mark.parametrize("dynamic", [True, False])
def test_clover_mat_and_matpc(prec, dynamic):
    X = (4, 4, 6, 4)
    P = Problem(X, prec, 12, CudaMem, clover=True, compressed=dynamic, dynamic=dynamic)
    full = P.spinor(seed=3, nparity=2)
    op = DR.Dirac("clover", P.U, KAPPA, clover=P.A, clover_inv=P.Ainv)
    for dagger in (0, 1):
        out = P.empty(2)
        op.M(out, P.to_dev(full, 2), dagger=dagger)
        assert_close(oracle.clover_mat(P.gauge, P.clover, full, X, KAPPA, dagger), P.to_host(out), prec, 12, "clover M")
    s = P.spinor(seed=4)
    for matpc in range(4):
        pc = DR.Dirac("cloverpc", P.U, KAPPA, clover=P.A, clover_inv=P.Ainv, matpc_type=matpc)
        for dagger in (0, 1):
            out = P.empty()
            pc.M(out, P.to_dev(s), dagger=dagger)
            ref = oracle.clover_matpc(P.gauge, P.clover, P.clover_inv, s, X, KAPPA, matpc, dagger)
            assert_close(ref, P.to_host(out), prec, 12, f"clover Mpc type={matpc} dag={dagger}")


def test_cg_wilson_double():
    P = Problem(X8, 8, 18, CudaMem)
    res, true_res, _, _ = solve(P, "wilsonpc", "cg")
    assert res.iter < 2000 and res.true_res < 5e-10
    assert true_res < 1e-8, true_res  # host-verified residual of the FULL system (normal-equation solve squares the condition)


def test_cg_clover_mixed_precision():
    """config 5 in miniature: clover, CG on MdagM, double precise / single sloppy with reliable updates"""
    P = Problem(X8, 8, 18, CudaMem, clover=True, compressed=True, dynamic=True)
    res, true_res, _, _ = solve(P, "cloverpc", "cg", mixed=True)
    assert res.reliable_updates >= 1
    assert res.true_res < 5e-10, res.true_res
    assert true_res < 1e-8, true_res


def test_partitioned_operators_through_cpp_layer():
    """DiracWilsonPC / DiracCloverPC with a (self-)partitioned lattice: the C++ layer drives pack + interior + exterior
    itself through its CommContext; results must equal the unpartitioned oracle."""
    from quda_b200 import comm
    X = (4, 6, 4, 8)
    P = Problem(X, 8, 12, CudaMem, clover=True, compressed=True, dynamic=True)
    ex = comm.HaloExchange(comm.ProcessGrid((1, 1, 1, 1), 0), X, 8, mode="self")
    cs = ex.comm_struct()
    s = P.spinor(seed=4)
    pc = DR.Dirac("wilsonpc", P.U, KAPPA, comm=cs)
    for dagger in (0, 1):
        out = P.empty()
        pc.M(out, P.to_dev(s), dagger=dagger)
        assert_close(oracle.wil_matpc(P.gauge, s, X, KAPPA, 0, dagger), P.to_host(out), 8, 12, "partitioned wilson Mpc")
    cpc = DR.Dirac("cloverpc", P.U, KAPPA, clover=P.A, comm=cs)
    for dagger in (0, 1):
        out = P.empty()
        cpc.M(out, P.to_dev(s), dagger=dagger)
        ref = oracle.clover_matpc(P.gauge, P.clover, P.clover_inv, s, X, KAPPA, 0, dagger)
        assert_close(ref, P.to_host(out), 8, 12, "partitioned clover Mpc")
    full = P.spinor(seed=5, nparity=2)
    op = DR.Dirac("wilson", P.U, KAPPA, comm=cs)
    out = P.empty(2)
    op.M(out, P.to_dev(full, 2))
    assert_close(oracle.wil_mat(P.gauge, full, X, KAPPA, 0), P.to_host(out), 8, 12, "partitioned wilson M")
    assert not ex.timed_out()


@pytest.mark.parametrize("prec", [8, 4])
def test_twisted_mass_mat_and_matpc(prec):
    """DiracTwistedMass / DiracTwistedMassPC (lib/dirac_twisted_mass.cpp) against tm_mat / tm_matpc"""
    X = (4, 6, 4, 8)
    P = Problem(X, prec, 12, CudaMem)
    full = P.spinor(seed=3, nparity=2)
    op = DR.Dirac("twistedmass", P.U, KAPPA, mu=MU)
    for dagger in (0, 1):
        out = P.empty(2)
        op.M(out, P.to_dev(full, 2), dagger=dagger)
        assert_close(oracle.tm_mat(P.gauge, full, X, KAPPA, MU, dagger), P.to_host(out), prec, 12, "twisted-mass M")
    s = P.spinor(seed=4)
    for matpc in range(4):
        pc = DR.Dirac("twistedmasspc", P.U, KAPPA, matpc_type=matpc, mu=MU)
        for dagger in (0, 1):
            out = P.empty()
            pc.M(out, P.to_dev(s), dagger=dagger)
            ref = oracle.tm_matpc(P.gauge, s, X, KAPPA, MU, matpc, dagger)
            assert_close(ref, P.to_host(out), prec, 12, f"twisted-mass Mpc type={matpc} dag={dagger}")


@pytest.mark.parametrize("matpc", [DR.MATPC_EVEN_EVEN, DR.MATPC_ODD_ODD_ASYMMETRIC])
def test_cg_twisted_mass_full_system(matpc):
    """prepare -> CG on MpcdagMpc -> reconstruct for the twisted-mass operator, verified with the oracle's tm_mat"""
    P = Problem(X8, 8, 18, CudaMem)
    res, true_res, _, _ = solve(P, "twistedmasspc", "cg", matpc)
    assert res.iter < 2000 and true_res < 1e-8, (res.iter, true_res)


@pytest.mark.parametrize("mixed", [False, True])
def test_cg_on_a_non_blocking_stream(mixed):
    """Every kernel of the operator / blas / solver layer must run on the operator's stream: build the operators on a
    cudaStreamNonBlocking stream (any torch side stream is one -- it does NOT synchronise with the legacy default stream)
    while the default stream is kept busy with unrelated work, and solve.  With blas kernels on the default stream (the
    round-1 bug) axpyNorm / reDotProduct would race against MdagM and the solve would diverge or return garbage."""
    P = Problem(X8, 8, 18, CudaMem, clover=True, compressed=True, dynamic=True)
    with busy_default_stream() as side:
        res, true_res, _, _ = solve(P, "cloverpc", "cg", mixed=mixed, stream=side.cuda_stream)
    assert res.iter < 2000 and res.true_res < 5e-10, (res.iter, res.true_res)
    assert true_res < 1e-8, true_res
    # the host followed the GPU one iteration behind: about one stream synchronisation per iteration, none of them on
    # the critical path (the reference's CG has two blocking reductions per iteration, lib/inv_cg_quda.cpp:354-377)
    assert res.host_syncs <= res.iter + 4 * (res.reliable_updates + 2), (res.host_syncs, res.iter, res.reliable_updates)


def test_reductions_are_bit_reproducible():
    """two-stage reductions summed in a fixed order: the same solve twice gives bit-identical iteration counts and
    residuals (the reference needs QUDA_DETERMINISTIC_REDUCE for this, include/communicator_quda.h:570)"""
    P = Problem(X8, 8, 18, CudaMem)
    a = solve(P, "wilsonpc", "cg")
    b = solve(P, "wilsonpc", "cg")
    assert a[0].iter == b[0].iter and a[0].true_res == b[0].true_res and a[1] == b[1]
