"""CPU tier: operator-level parity of the product's site code (host twin) against the oracle:
xpay / dagger / full fields, clover (compressed + dynamic Cholesky, uncompressed + static inverse),
self-partitioned halo (pack + interior + fused exterior) for all 16 partition masks."""
import itertools

import pytest

import ops
from common import HostMem, twin_backend


@pytest.mark.parametrize("prec", [8, 4, 2])
@pytest.mark.parametrize("recon", [18, 12, 8])
def test_xpay_dagger_fullfield(prec, recon):
    ops.check_xpay_fullfield(HostMem, twin_backend(), prec, recon)


@pytest.mark.parametrize("prec", [8, 4, 2])
@pytest.mark.parametrize("compressed,dynamic", [(True, True), (False, True), (False, False), (True, False)])
def test_clover(prec, compressed, dynamic):
    ops.check_clover(HostMem, twin_backend(), prec, 12, compressed, dynamic)


MASKS = [tuple((m >> d) & 1 for d in range(4)) for m in range(1, 16)]


@pytest.mark.parametrize("comm_dim", MASKS)
def test_partitioned_wilson_all_masks(comm_dim):
    ops.check_partitioned(HostMem, twin_backend(), 8, 18, comm_dim, X=(4, 6, 4, 8))


@pytest.mark.parametrize("prec,recon", [(8, 12), (4, 12), (4, 8), (2, 18), (2, 8)])
@pytest.mark.parametrize("comm_dim", [(1, 0, 0, 0), (0, 0, 0, 1), (1, 1, 1, 1)])
def test_partitioned_wilson_precisions(prec, recon, comm_dim):
    ops.check_partitioned(HostMem, twin_backend(), prec, recon, comm_dim, xpay=True, dagger=1)


@pytest.mark.parametrize("op", ["clover_pc", "clover"])
@pytest.mark.parametrize("prec", [8, 2])
@pytest.mark.parametrize("comm_dim", [(0, 1, 0, 1), (1, 1, 1, 1)])
def test_partitioned_clover(op, prec, comm_dim):
    ops.check_partitioned(HostMem, twin_backend(), prec, 12, comm_dim, op=op, xpay=True,
                          clover_kw=dict(compressed=True, dynamic=True))


@pytest.mark.parametrize("comm_dim", MASKS)
def test_partitioned_reference_style_split(comm_dim):
    """explicit INTERIOR (masked partial sums) + EXTERIOR (read-modify-write) kernels, the reference's decomposition"""
    ops.check_partitioned(HostMem, twin_backend(), 8, 12, comm_dim, X=(4, 6, 4, 8), xpay=True, split=True)


@pytest.mark.parametrize("op", ["wilson", "clover_pc", "clover"])
@pytest.mark.parametrize("tile", [(16, 2, 2, 1), (2, 2, 2, 2), (1, 4, 1, 2), (2, 8, 4, 2)])
@pytest.mark.parametrize("comm_dim", [(0, 0, 0, 1), (0, 1, 1, 1), (1, 1, 1, 1), (1, 0, 1, 0)])
def test_boundary_slab_schedule(op, tile, comm_dim):
    """interior tile box + boundary slabs must cover every site exactly once for any tiling / partition mask
    (including tilings with 1 or 2 tiles along a partitioned dimension)"""
    ops.check_partitioned(HostMem, twin_backend(), 8, 18, comm_dim, op=op, X=(8, 6, 4, 8), xpay=True, tile=tile,
                          clover_kw=dict(compressed=True, dynamic=True))


@pytest.mark.parametrize("comm_dim", [(0, 0, 0, 1), (0, 1, 1, 1), (1, 1, 1, 1)])
@pytest.mark.parametrize("op", ["wilson", "clover_pc"])
def test_boundary_and_interior_tiles_are_independent(op, comm_dim):
    """BOUNDARY_TILES and INTERIOR_TILES launches write disjoint sites, in any order (they run on different streams)"""
    ops.check_partitioned(HostMem, twin_backend(), 4, 12, comm_dim, op=op, X=(8, 6, 4, 8), xpay=True, split="tiles",
                          clover_kw=dict(compressed=True, dynamic=True))


@pytest.mark.parametrize("prec,recon", [(8, 18), (8, 12), (4, 12), (4, 8), (2, 12), (2, 8)])
@pytest.mark.parametrize("n_src", [2, 5, 8])
@pytest.mark.parametrize("flavour", ["thread", "auto"])
def test_multi_rhs_wilson(monkeypatch, prec, recon, n_src, flavour):
    """batched Dslash (cvector_ref form): in-thread batches of 4 / 2 + single-source tail ("thread"), and whatever
    the library picks by default for the precision ("auto")"""
    monkeypatch.setenv("B200_MRHS_MODE", flavour)
    ops.check_multi_rhs(HostMem, twin_backend(), prec, recon, n_src, xpay=(n_src == 5), dagger=n_src % 2)


@pytest.mark.parametrize("op", ["clover_pc", "clover"])
@pytest.mark.parametrize("prec", [8, 4, 2])
def test_multi_rhs_clover(monkeypatch, op, prec):
    monkeypatch.setenv("B200_MRHS_MODE", "thread")
    ops.check_multi_rhs(HostMem, twin_backend(), prec, 12, 3, op=op, xpay=True)


def test_multi_rhs_full_fields_and_fallback():
    be = twin_backend()
    ops.check_multi_rhs(HostMem, be, 4, 12, 4, xpay=True, nparity=2)                     # full fields (both parities)
    ops.check_multi_rhs(HostMem, be, 8, 18, 1, comm_dim=(1, 0, 0, 1), X=(4, 4, 4, 4))    # partitioned -> per-source path


def test_multi_rhs_argument_checks():
    from common import Problem
    from quda_b200 import dslash as D
    from quda_b200.lib import B200Error
    be = twin_backend()
    P = Problem((4, 4, 4, 4), 4, 12, HostMem)
    ins = [P.to_dev(P.spinor(seed=i)) for i in range(3)]
    outs = [P.empty() for _ in range(3)]
    with pytest.raises(B200Error, match="aliases"):
        D.ApplyWilson([outs[0], outs[0], outs[2]], ins, P.U, 0.0, None, 0, 0, backend=be)
    with pytest.raises(B200Error, match="aliases"):
        D.ApplyWilson([outs[0], ins[2], outs[2]], ins, P.U, 0.0, None, 0, 0, backend=be)
    with pytest.raises(B200Error, match="n_src"):
        D.ApplyWilson([P.empty() for _ in range(17)], [ins[0]] * 17, P.U, 0.0, None, 0, 0, backend=be)
    with pytest.raises(B200Error, match="x is null"):
        D.ApplyWilson(outs, ins, P.U, -0.1, None, 0, 0, backend=be)


@pytest.mark.parametrize("prec,recon", [(8, 18), (4, 12), (4, 8), (2, 12), (2, 18)])
@pytest.mark.parametrize("n_src,cta_sources", [(2, 0), (5, 2), (8, 0), (16, 3)])
def test_multi_rhs_cta_flavour(monkeypatch, prec, recon, n_src, cta_sources):
    """B200_MRHS_MODE=cta: one thread per (site, source), sources of a site share a CTA; ragged last batch included"""
    monkeypatch.setenv("B200_MRHS_MODE", "cta")
    monkeypatch.setenv("B200_MRHS_CTA_SOURCES", str(cta_sources))
    ops.check_multi_rhs(HostMem, twin_backend(), prec, recon, n_src, xpay=(n_src == 5), dagger=n_src % 2,
                        tile=(2, 2, 2, 1))


def test_multi_rhs_cta_flavour_clover_and_full(monkeypatch):
    monkeypatch.setenv("B200_MRHS_MODE", "cta")
    be = twin_backend()
    ops.check_multi_rhs(HostMem, be, 4, 12, 3, op="clover_pc", xpay=True)
    ops.check_multi_rhs(HostMem, be, 2, 12, 3, op="clover", xpay=True, tile=(2, 2, 1, 1))
    ops.check_multi_rhs(HostMem, be, 4, 12, 4, xpay=True, nparity=2, tile=(2, 2, 2, 2))


@pytest.mark.parametrize("prec,recon", [(8, 18), (8, 12), (4, 12), (4, 8), (2, 18), (2, 12)])
def test_twisted_mass(prec, recon):
    """degenerate twisted mass: ApplyTwistedMass / ApplyTwistedMassPreconditioned + the PC operator composition"""
    ops.check_twisted_mass(HostMem, twin_backend(), prec, recon)


@pytest.mark.parametrize("comm_dim", [(0, 0, 0, 1), (1, 1, 1, 1)])
@pytest.mark.parametrize("prec", [8, 2])
def test_twisted_mass_partitioned(prec, comm_dim):
    ops.check_twisted_mass(HostMem, twin_backend(), prec, 12, X=(4, 4, 4, 4), comm_dim=comm_dim)


def test_twisted_mass_argument_checks():
    from common import Problem
    from quda_b200 import dslash as D
    from quda_b200.lib import B200Error
    be = twin_backend()
    P = Problem((4, 4, 4, 4), 4, 12, HostMem)
    s, out = P.to_dev(P.spinor(seed=1)), P.empty()
    with pytest.raises(B200Error, match="only defined for xpay"):
        D.ApplyTwistedMass(out, s, P.U, 0.0, 0.1, s, 0, 0, backend=be)
    with pytest.raises(B200Error, match="only defined for dagger"):
        D.ApplyTwistedMassPreconditioned(out, s, P.U, 1.0, 0.1, False, None, 0, 0, True, backend=be)
    with pytest.raises(B200Error, match="not defined for xpay"):
        D.ApplyTwistedMassPreconditioned(out, s, P.U, 1.0, 0.1, True, P.to_dev(P.spinor(seed=2)), 0, 1, True, backend=be)
    h = ops.self_halo(P, HostMem, (0, 0, 0, 1))
    with pytest.raises(B200Error, match="pack kernel"):
        D.ApplyTwistedMassPreconditioned(out, s, P.U, 1.0, 0.1, False, None, 0, 1, False, halo=h, backend=be)


@pytest.mark.parametrize("split", ["fused", "fused_roles"])
@pytest.mark.parametrize("comm_dim", MASKS)
def test_fused_single_launch_all_masks(comm_dim, split):
    """b200_dslash_apply_fused (pack + interior + boundary as one launch, or its pack + boundary and interior roles as two):
    the interior role (every tile, face sites retire) and the boundary role (one thread per face site, corners owned by
    the highest partitioned dimension) must cover every site exactly once and reproduce the periodic operator for all
    15 partition masks"""
    ops.check_partitioned(HostMem, twin_backend(), 8, 18, comm_dim, X=(4, 6, 4, 8), split=split)


@pytest.mark.parametrize("prec,recon", [(4, 12), (2, 8)])
@pytest.mark.parametrize("op", ["wilson", "clover_pc"])
def test_fused_single_launch_ops(prec, recon, op):
    ops.check_partitioned(HostMem, twin_backend(), prec, recon, (1, 0, 1, 1), op=op, xpay=(op == "wilson"), dagger=1, split="fused",
                          X=(8, 4, 4, 6))


@pytest.mark.parametrize("comm_dim", MASKS)
def test_site_granular_split_all_masks(comm_dim):
    """B200_KERNEL_BOUNDARY_SITES + B200_KERNEL_INTERIOR_SITES (what the operator layer puts on its side / main stream):
    together they update every site exactly once for all 15 partition masks"""
    ops.check_partitioned(HostMem, twin_backend(), 4, 12, comm_dim, X=(4, 6, 4, 8), split="sites", xpay=True)


# ---- batched (multi-RHS) halo: one pack launch for all sources, one arrival signal per face (b200_pack_ghost_multi)
@pytest.mark.parametrize("comm_dim", MASKS)
def test_batched_halo_all_masks(comm_dim):
    ops.check_partitioned_multi(HostMem, twin_backend(), 8, 18, comm_dim, 3, X=(4, 6, 4, 8), xpay=True)


@pytest.mark.parametrize("prec,recon", [(8, 12), (4, 12), (4, 8), (2, 18), (2, 12)])
@pytest.mark.parametrize("n_src,aligned", [(1, True), (2, False), (5, True), (16, False)])
def test_batched_halo_precisions(prec, recon, n_src, aligned):
    ops.check_partitioned_multi(HostMem, twin_backend(), prec, recon, (1, 0, 1, 1), n_src, dagger=1, aligned=aligned)


@pytest.mark.parametrize("op", ["clover_pc", "clover"])
@pytest.mark.parametrize("split", [None, "tiles", "sites"])
def test_batched_halo_ops_and_schedules(op, split):
    ops.check_partitioned_multi(HostMem, twin_backend(), 4, 12, (0, 1, 1, 1), 4, op=op, xpay=True, split=split,
                                clover_kw=dict(compressed=True, dynamic=True))


@pytest.mark.parametrize("flavour", ["thread", "cta"])
@pytest.mark.parametrize("prec,recon,n_src", [(8, 18, 5), (4, 12, 7), (2, 8, 4)])
def test_batched_halo_batched_interior_flavours(monkeypatch, flavour, prec, recon, n_src):
    """on a partitioned lattice the interior tiles of a batch run through the multi-RHS kernels (both flavours; odd
    sources out through the single-source kernel), the boundary tiles per source -- the lattice must be covered exactly once"""
    monkeypatch.setenv("B200_MRHS_MODE", flavour)
    ops.check_partitioned_multi(HostMem, twin_backend(), prec, recon, (0, 1, 0, 1), n_src, X=(8, 8, 4, 8), xpay=True)
    ops.check_partitioned_multi(HostMem, twin_backend(), prec, recon, (0, 0, 1, 1), n_src, X=(4, 4, 8, 6), split="tiles")


def test_batched_halo_arrival_protocol():
    """the ticket protocol of the batched pack (host-twin CTA walk in scrambled order): every face's arrival counter moves
    exactly once, after all sources have landed, to the value a single exchange `seq` would publish"""
    import ctypes as C
    import numpy as np
    from quda_b200 import dslash as D, fields as F, lib as L
    from common import Problem
    be = twin_backend()
    X, prec, n_src = (4, 6, 4, 8), 4, 3
    P = Problem(X, prec, 12, HostMem)
    ins = [P.to_dev(P.spinor(seed=70 + i)) for i in range(n_src)]
    flags = np.zeros(8, dtype=np.uint32)
    counters = np.zeros(8, dtype=np.int32)
    comm_dim = (1, 0, 1, 1)
    for seq in (1, 2, 3, 4):
        a = L.PackArgs()
        a.abi_version, a.precision = L.ABI_VERSION, prec
        bufs = []
        stride = (C.c_size_t * 4)()
        for d in range(4):
            a.X[d], a.comm_dim[d] = X[d], comm_dim[d]
            stride[d] = F.ghost_parity_bytes(X, prec, d)
            for f in range(2):
                if comm_dim[d]:
                    bufs.append(np.zeros(n_src * stride[d], dtype=np.uint8))
                    a.dst[d][f] = bufs[-1].ctypes.data
                    a.signal[d][f] = flags.ctypes.data + 4 * (2 * d + f)
        a.block_counter = counters.ctypes.data
        a.seq, a.parity, a.dagger = seq, 0, 0
        a.in_ = ins[0].desc()
        srcs = (L.Spinor * n_src)(*[f.desc() for f in ins])
        be.call("pack_ghost_multi", C.byref(a), n_src, srcs, stride)
        uses = (seq + (seq & 1)) // 2
        for d in range(4):
            face_cb = F.volume_cb(X) // X[d]
            for f in range(2):
                assert flags[2 * d + f] == (uses * face_cb if comm_dim[d] else 0)
        assert not counters.any()


def test_batched_halo_argument_checks():
    import ctypes as C
    from quda_b200 import lib as L
    from common import Problem
    be = twin_backend()
    P = Problem((4, 4, 4, 4), 4, 12, HostMem)
    f = P.to_dev(P.spinor())
    a = L.PackArgs()
    a.abi_version, a.precision = L.ABI_VERSION, 4
    buf = HostMem.empty(1 << 16)
    for d in range(4):
        a.X[d], a.comm_dim[d] = 4, 1
        for k in range(2):
            a.dst[d][k] = buf.ctypes.data
    srcs = (L.Spinor * 2)(f.desc(), f.desc())
    small = (C.c_size_t * 4)(8, 8, 8, 8)
    with pytest.raises(L.B200Error, match="smaller than one face"):
        be.call("pack_ghost_multi", C.byref(a), 2, srcs, small)
    odd = (C.c_size_t * 4)(4104, 4104, 4104, 4104)
    with pytest.raises(L.B200Error, match="multiple of 16"):
        be.call("pack_ghost_multi", C.byref(a), 2, srcs, odd)
    ok = (C.c_size_t * 4)(4096, 4096, 4096, 4096)
    with pytest.raises(L.B200Error, match="n_src"):
        be.call("pack_ghost_multi", C.byref(a), 17, srcs, ok)
    with pytest.raises(L.B200Error, match="n_src"):
        be.call("pack_ghost_multi", C.byref(a), 0, srcs, ok)
    # a batch on a partitioned lattice needs one ghost slab per source: src_stride 0 (all sources on slab 0) is refused
    from quda_b200 import dslash as D
    import ops
    halo = ops.self_halo(P, HostMem, (0, 0, 0, 1))
    outs, ins = [P.empty(), P.empty()], [f, P.to_dev(P.spinor(seed=3))]
    with pytest.raises(L.B200Error, match="own ghost slab"):
        D.ApplyWilson(outs, ins, P.U, 0.0, None, 0, 0, halo=halo, backend=be)
    # the fused Dslash refuses pack arguments that do not describe its own input's faces
    dst = [[None, None]] * 3 + [[halo.ghost[3][1], halo.ghost[3][0]]]
    fused = dict(halo=halo, fused_dst=dst, block_counter=HostMem.empty(32))

    def tampered(edit):  # the twin, with the pack arguments edited on the way in
        class Backend:
            def call(self, name, args, pack):
                edit(pack._obj)
                return be.call(name, args, pack)
        return Backend()
    D.ApplyWilson(outs[0], f, P.U, 0.0, None, 0, 0, backend=be, **fused)
    with pytest.raises(L.B200Error, match="kernel must be AUTO"):
        D.ApplyWilson(outs[0], f, P.U, 0.0, None, 0, 0, backend=be, kernel=L.KERNEL_INTERIOR, **fused)
    with pytest.raises(L.B200Error, match=r"dst\[3\]\[1\] is NULL"):
        D.ApplyWilson(outs[0], f, P.U, 0.0, None, 0, 0, backend=be, **dict(fused, fused_dst=dst[:3] + [[dst[3][0], None]]))
    with pytest.raises(L.B200Error, match="different sequence numbers"):
        D.ApplyWilson(outs[0], f, P.U, 0.0, None, 0, 0, backend=tampered(lambda p: setattr(p, "seq", p.seq + 1)), **fused)
    with pytest.raises(L.B200Error, match="extents differ"):
        D.ApplyWilson(outs[0], f, P.U, 0.0, None, 0, 0, backend=tampered(lambda p: p.X.__setitem__(0, 8)), **fused)


@pytest.mark.parametrize("prec,recon,n_src,dims", [(8, 18, 3, (0, 0, 0, 1)), (4, 12, 8, (0, 1, 1, 1)), (2, 12, 4, (1, 1, 1, 1))])
def test_batched_exchange_schedule_with_arrival_counters(prec, recon, n_src, dims):
    """HaloExchange(mode="self", n_src=...) end to end on the CPU stand-in: batched and single exchanges interleaved on the
    same double-buffered slabs; the twin refuses to run a boundary role whose arrival counter is below its target"""
    import numpy as np
    import oracle
    from common import Problem, assert_close, host_self_exchange
    from quda_b200 import comm
    X = (8, 4, 4, 8)
    P = Problem(X, prec, recon, HostMem)
    ex = host_self_exchange(X, prec, dims, n_src)
    src = [P.spinor(seed=10 + i) for i in range(n_src)]
    dins, outs, one = [P.to_dev(s) for s in src], [P.empty() for _ in range(n_src)], P.empty()
    for rep in range(5):
        comm.apply_wilson_distributed(ex, outs, dins, P.U, 0.0, None, 0, 0)
        if rep % 2:
            comm.apply_wilson_distributed(ex, one, dins[1], P.U, 0.0, None, 0, 0)
    for i in range(n_src):
        assert_close(oracle.wil_dslash(P.gauge, src[i], X, 0, 0), P.to_host(outs[i]), prec, recon, f"batched self exchange src {i}")
    assert np.array_equal(P.to_host(one), P.to_host(outs[1]))
    assert ex.seq == 7 and not ex.timed_out()
    with pytest.raises(Exception, match="batch of"):
        ex.start(dins + dins[:1], 1, 0)


def test_twin_refuses_a_halo_that_never_arrives():
    """negative control of the check above: a Dslash whose exchange number is ahead of the counters is an error"""
    from common import Problem, host_self_exchange
    from quda_b200 import comm, dslash as D, lib as L
    X = (4, 4, 4, 8)
    P = Problem(X, 4, 12, HostMem)
    ex = host_self_exchange(X, 4, (0, 0, 0, 1))
    din, out = P.to_dev(P.spinor()), P.empty()
    comm.apply_wilson_distributed(ex, out, din, P.U, 0.0, None, 0, 0)
    h = ex.halo()
    h.seq += 2  # same buffer, one exchange later: nobody has packed it
    with pytest.raises(L.B200Error, match="never finish"):
        D.ApplyWilson(out, din, P.U, 0.0, None, 0, 0, halo=comm._RawHalo(h), backend=twin_backend())


# ---- smallest / ragged local lattices (extent 2 is the smallest even extent; a partitioned dimension needs >= 4)
@pytest.mark.parametrize("X", [(2, 2, 2, 2), (4, 2, 2, 2), (2, 4, 6, 2), (6, 2, 2, 10)])
def test_minimal_and_ragged_lattices(X):
    be = twin_backend()
    ops.check_xpay_fullfield(HostMem, be, 8, 18, X=X)
    ops.check_xpay_fullfield(HostMem, be, 2, 12, X=X)
    for d in range(4):
        mask = tuple(int(e == d) for e in range(4))
        if X[d] >= 4:
            for split in (False, "tiles", "sites", "fused", "fused_roles"):
                ops.check_partitioned(HostMem, be, 4, 12, mask, X=X, xpay=True, split=split)
        else:
            from quda_b200 import lib as L
            with pytest.raises(L.B200Error, match="needs local extent >= 4"):
                ops.check_partitioned(HostMem, be, 4, 12, mask, X=X)
