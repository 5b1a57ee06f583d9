"""Parity cases shared by the CPU tier (host twin) and the GPU tier (libquda_b200.so): every case body runs once per tier,
with the memory class and the backend of that tier.  OPS is the one table of the operators they apply (entry point,
clover field, oracle reference), SPLITS the one table of the launches a halo split issues."""
import itertools
from typing import Callable, NamedTuple, Optional

import numpy as np

import oracle
from common import Problem, assert_close
from quda_b200 import dslash as D
from quda_b200 import fields as F
from quda_b200 import lib as L

KAPPA, MU = 0.12195, 0.1


def clover_inverse(P):
    """the clover field A^-1 is taken from: A itself under a dynamic inverse, the stored inverse under a static one"""
    return P.A if P.dynamic else P.Ainv


class Op(NamedTuple):
    entry: Callable                    # its D.Apply* entry point
    clover: Optional[Callable]         # P -> the clover field it reads (None: no clover term)
    dslash: Callable                   # (P, psi, parity, dagger) -> the oracle's D psi (A^-1 D psi for clover_pc)
    x_term: Callable                   # (P, x, parity, dagger) -> the oracle's x' of the xpay form x' + a D psi
    xpay_only: bool                    # the operator exists only in its xpay form


def _wil_dslash(P, psi, parity, dagger):
    return oracle.wil_dslash(P.gauge, psi, P.X, parity, dagger)


OPS = {
    "wilson": Op(D.ApplyWilson, None, _wil_dslash, lambda P, x, parity, dagger: x, False),
    "clover": Op(D.ApplyWilsonClover, lambda P: P.A, _wil_dslash,
                 lambda P, x, parity, dagger: oracle.apply_clover(P.clover, x, P.X, parity), True),
    "clover_pc": Op(D.ApplyWilsonCloverPreconditioned, clover_inverse,
                    lambda P, psi, parity, dagger: oracle.clover_dslash(P.gauge, P.clover_inv, psi, P.X, parity, dagger),
                    lambda P, x, parity, dagger: x, False),
    "tm": Op(D.ApplyTwistedMass, None, _wil_dslash,
             lambda P, x, parity, dagger: oracle.twist_gamma5(x, KAPPA, MU, dagger), True),
}


def takes_x(op, xpay):
    """whether a case of `op` runs its xpay form x' + a D psi"""
    return xpay or OPS[op].xpay_only


def apply(P, op, out, in_, a, x, parity, dagger, **kw):
    """`op` through its entry point on the fields of P (a Problem or a precise_cases.Fields); out / in_ / x may be lists
    of fields (a multi-RHS batch).  kw go to the entry point: backend, halo, kernel, tile, ... and b, the twist of tm."""
    row = OPS[op]
    A = (row.clover(P),) if row.clover else ()
    row.entry(out, in_, P.U, *A, a=a, x=x, parity=parity, dagger=dagger, **kw)


def reference(P, op, psi, parity, dagger, x=None, a=0.0):
    """the oracle's `op` on one parity in float64: D psi, or x' + a D psi with x' = x (A x for clover, the twisted x for
    tm) when x is given"""
    row = OPS[op]
    d = row.dslash(P, psi, parity, dagger).astype(np.float64)
    return d if x is None else xpay(row.x_term(P, x, parity, dagger), a, d)


def xpay(x, a, d):
    """x + a d in float64"""
    return x.astype(np.float64) + a * d.astype(np.float64)


def full_dslash(P, full, dagger):
    """the oracle's D on a full field [even | odd]: each parity from the other parity's sites"""
    return np.concatenate([oracle.wil_dslash(P.gauge, full[P.Vh:], P.X, 0, dagger),
                           oracle.wil_dslash(P.gauge, full[:P.Vh], P.X, 1, dagger)])


# split name -> the launches one application issues (the default None: one AUTO launch)
SPLITS = {
    None: [dict()],
    # the two halves of AUTO issued separately (boundary first: they are independent)
    "tiles": [dict(kernel=L.KERNEL_BOUNDARY_TILES), dict(kernel=L.KERNEL_INTERIOR_TILES)],
    # the same split with 1-site-thick shells
    "sites": [dict(kernel=L.KERNEL_BOUNDARY_SITES), dict(kernel=L.KERNEL_INTERIOR_SITES)],
    # reference-style: masked INTERIOR then EXTERIOR read-modify-write
    "reference": [dict(kernel=L.KERNEL_INTERIOR), dict(kernel=L.KERNEL_EXTERIOR)],
    # pack + interior + boundary in one call (b200_dslash_apply_fused)
    "fused": [dict()],
    # the fused launch's roles as the `split` halo schedule issues them: pack + boundary, then the interior
    "fused_roles": [dict(kernel=L.KERNEL_BOUNDARY_TILES), dict(kernel=L.KERNEL_INTERIOR_TILES)],
}


def wilson_vs_oracle(P, be, s, parity, dagger, what, **kw):
    """D s on one parity through ApplyWilson against the oracle; returns the deviation"""
    out = P.empty()
    D.ApplyWilson(out, P.to_dev(s), P.U, 0.0, None, parity, dagger, backend=be, **kw)
    return assert_close(oracle.wil_dslash(P.gauge, s, P.X, parity, dagger), P.to_host(out), P.prec, P.recon, what)


def check_wilson_dslash(mem, be, prec, recon, X):
    """D on single-parity fields for both parities and daggers; returns the worst deviation"""
    P = Problem(X, prec, recon, mem)
    return max(wilson_vs_oracle(P, be, P.spinor(seed=11 + parity), parity, dagger, f"X={X} parity={parity} dagger={dagger}")
               for parity in (0, 1) for dagger in (0, 1))


def check_tma_work_ranges(mem, be, env, links, grid):
    """both link modes (-1: register stream, 0 / n: shared-memory stages) and every work partition (ranges that start / end
    mid-tile, one item per CTA, one CTA for everything): no deadlock, no slot hazard, every site visited once"""
    env.setenv("B200_TMA_LINKS", str(links))
    env.setenv("B200_TMA_GRID", str(grid))
    P = Problem((16, 4, 8, 6), 4, 12, mem, anisotropy=1.7)
    wilson_vs_oracle(P, be, P.spinor(seed=5), 1, 0, f"links={links} grid={grid}")


def check_tma_register_stream_links(mem, be, env, prefetch, rings, grid):
    """register-stream links: every prefetch distance (the reload of a direction pair targets this item or the next one)
    and spinor ring depth, with work ranges that cross tiles and parities (full field)"""
    env.setenv("B200_TMA_LINKS", "-1")
    env.setenv("B200_TMA_PREFETCH", str(prefetch))
    env.setenv("B200_TMA_RINGS", rings)
    env.setenv("B200_TMA_GRID", str(grid))
    P = Problem((8, 4, 4, 6), 4, 12, mem)
    full = P.spinor(seed=3, nparity=2)
    out = P.empty(2)
    D.ApplyWilson(out, P.to_dev(full, 2), P.U, 0.0, None, D.QUDA_INVALID_PARITY, 1, backend=be)
    assert_close(full_dslash(P, full, 1), P.to_host(out), 4, 12, f"prefetch={prefetch} rings={rings}")


def check_tma_l2_prefetch_lookahead(mem, be, env, l2pf):
    """the L2 prefetch of the link boxes is a hint (no functional effect) but its coordinates come from the same box
    function: every look-ahead, including one beyond the end of a CTA's work range, must leave the result unchanged"""
    env.setenv("B200_TMA_L2PF", str(l2pf))
    env.setenv("B200_TMA_GRID", "7")
    P = Problem((16, 4, 4, 6), 4, 12, mem)
    wilson_vs_oracle(P, be, P.spinor(seed=8), 0, 0, f"l2pf={l2pf}")


def check_tma_tiles(mem, be, env, tile):
    """tile shapes incl. TY == 1 / TZ == 1 (the backward y / z links then come from one box only) and a tile that
    spans the whole extent (the halo rows are the tile's own opposite edge)"""
    env.setenv("B200_TMA_TILE", tile)
    P = Problem((8, 8, 4, 4), 4, 12, mem)
    s = P.spinor(seed=6)
    for parity in (0, 1):
        wilson_vs_oracle(P, be, s, parity, 1, f"tile {tile} parity {parity}")


def check_xpay_fullfield(mem, be, prec, recon, X=(4, 6, 4, 8)):
    P = Problem(X, prec, recon, mem, anisotropy=1.3)
    s, xs = P.spinor(seed=3), P.spinor(seed=4)
    for parity, dagger in itertools.product((0, 1), (0, 1)):
        out = P.empty()
        apply(P, "wilson", out, P.to_dev(s), -KAPPA, P.to_dev(xs), parity, dagger, backend=be)
        assert_close(reference(P, "wilson", s, parity, dagger, xs, -KAPPA), P.to_host(out), prec, recon,
                     f"xpay p={parity} dag={dagger}")
    full = P.spinor(seed=9, nparity=2)
    for dagger in (0, 1):
        out, inp = P.empty(2), P.to_dev(full, 2)
        D.ApplyWilson(out, inp, P.U, -KAPPA, inp, D.QUDA_INVALID_PARITY, dagger, backend=be)
        assert_close(oracle.wil_mat(P.gauge, full, X, KAPPA, dagger), P.to_host(out), prec, recon, "full-field M")
        out2 = P.empty(2)
        D.ApplyWilson(out2, inp, P.U, 0.0, None, D.QUDA_INVALID_PARITY, dagger, backend=be)
        assert_close(full_dslash(P, full, dagger), P.to_host(out2), prec, recon, "full-field D")


def check_clover(mem, be, prec, recon, compressed, dynamic, X=(4, 4, 6, 4)):
    P = Problem(X, prec, recon, mem, clover=True, compressed=compressed, dynamic=dynamic)
    s, xs = P.spinor(seed=21), P.spinor(seed=22)
    for parity in (0, 1):
        # ApplyClover: A x and A^{-1} x
        out = P.empty()
        D.ApplyClover(out, P.to_dev(s), P.A, False, parity, backend=be)
        assert_close(oracle.apply_clover(P.clover, s, X, parity), P.to_host(out), prec, recon, "ApplyClover A")
        out = P.empty()
        D.ApplyClover(out, P.to_dev(s), clover_inverse(P), True, parity, backend=be)
        assert_close(oracle.apply_clover(P.clover_inv, s, X, parity), P.to_host(out), prec, recon, "ApplyClover Ainv")
        for dagger in (0, 1):
            # preconditioned: A^{-1} D in
            out = P.empty()
            apply(P, "clover_pc", out, P.to_dev(s), 0.0, None, parity, dagger, backend=be)
            assert_close(reference(P, "clover_pc", s, parity, dagger), P.to_host(out), prec, recon,
                         f"clover-pc p={parity} dag={dagger}")
            # unpreconditioned xpay form: A x + a D in
            out = P.empty()
            apply(P, "clover", out, P.to_dev(s), -KAPPA, P.to_dev(xs), parity, dagger, backend=be)
            assert_close(reference(P, "clover", s, parity, dagger, xs, -KAPPA), P.to_host(out), prec, recon,
                         f"clover xpay p={parity} dag={dagger}")
        # x + a A^{-1} D in (no dagger)
        out = P.empty()
        apply(P, "clover_pc", out, P.to_dev(s), -KAPPA * KAPPA, P.to_dev(xs), parity, 0, backend=be)
        assert_close(reference(P, "clover_pc", s, parity, 0, xs, -KAPPA * KAPPA), P.to_host(out), prec, recon,
                     "clover-pc xpay")


def check_twisted_mass(mem, be, prec, recon, X=(4, 6, 4, 8), comm_dim=None):
    """Degenerate twisted mass: ApplyTwistedMass / ApplyTwistedMassPreconditioned and their composition into the
    even-odd preconditioned operator for all four matpc types (lib/dirac_twisted_mass.cpp:47-237) against the oracle's
    tm_dslash / tm_mat / tm_matpc (tests/host_reference/wilson_dslash_reference.cpp:139-315)."""
    P = Problem(X, prec, recon, mem)
    kappa, mu = KAPPA, MU
    s, xs = P.spinor(seed=41), P.spinor(seed=42)
    b_tw = 2 * mu * kappa                 # direct twist
    a_inv = -2.0 * kappa * mu             # inverse twist
    scale = 1.0 / (1.0 + a_inv * a_inv)

    def halo_for(field, in_parity, dagger):
        if comm_dim is None:
            return None
        h = self_halo(P, mem, comm_dim)
        self_exchange(P, h, field, in_parity, dagger, be)
        return h

    for parity, dagger in itertools.product((0, 1), (0, 1)):
        din = P.to_dev(s)
        # ApplyTwistedMass: a D in + (1 + i b gamma5) x
        out = P.empty()
        apply(P, "tm", out, din, -kappa, P.to_dev(xs), parity, dagger, b=b_tw, halo=halo_for(din, 1 - parity, dagger),
              backend=be)
        assert_close(reference(P, "tm", s, parity, dagger, xs, -kappa), P.to_host(out), prec, recon,
                     f"ApplyTwistedMass p={parity} dag={dagger}")
        # ApplyTwistedMassPreconditioned as DiracTwistedMassPC::Dslash / DslashXpay call it
        for matpc in range(4):
            asym = matpc >= 2 and dagger
            if comm_dim is not None and dagger and not asym:
                continue  # needs the twist in the pack kernel (rejected with B200_ERR_UNSUPPORTED, checked elsewhere)
            out = P.empty()
            D.ApplyTwistedMassPreconditioned(out, din, P.U, scale, a_inv, False, None, parity, dagger, asym,
                                             halo=halo_for(din, 1 - parity, dagger), backend=be)
            ref = oracle.tm_dslash(P.gauge, s, X, kappa, mu, parity, dagger, matpc).astype(np.float64)
            assert_close(ref, P.to_host(out), prec, recon, f"tm_dslash matpc={matpc} p={parity} dag={dagger}")
            if not asym:
                k = -kappa * kappa
                out = P.empty()
                D.ApplyTwistedMassPreconditioned(out, din, P.U, k * scale, a_inv, True, P.to_dev(xs), parity, dagger, False,
                                                 halo=halo_for(din, 1 - parity, dagger), backend=be)
                assert_close(xpay(xs, k, ref), P.to_host(out), prec, recon, f"tm_dslash xpay matpc={matpc} dag={dagger}")
    if comm_dim is not None:
        return
    # ApplyTwistGamma: the site-local rotation and its inverse
    for dagger, inverse in itertools.product((0, 1), (False, True)):
        out = P.empty()
        D.ApplyTwistGamma(out, P.to_dev(s), kappa, mu, dagger, inverse, backend=be)
        assert_close(oracle.twist_gamma5(s, kappa, mu, dagger, inverse), P.to_host(out), prec, 18, f"twist dag={dagger} inv={inverse}")
    # composition: DiracTwistedMassPC::M
    for matpc, dagger in itertools.product(range(4), (0, 1)):
        this = 0 if matpc in (0, 2) else 1
        other = 1 - this
        asym = matpc >= 2 and dagger
        din, tmp, out = P.to_dev(s), P.empty(), P.empty()
        D.ApplyTwistedMassPreconditioned(tmp, din, P.U, scale, a_inv, False, None, other, dagger, asym, backend=be)
        k2 = -kappa * kappa
        if matpc < 2:
            D.ApplyTwistedMassPreconditioned(out, tmp, P.U, k2 * scale, a_inv, True, din, this, dagger, False, backend=be)
        else:
            D.ApplyTwistedMass(out, tmp, P.U, k2, b_tw, din, this, dagger, backend=be)
        ref = oracle.tm_matpc(P.gauge, s, X, kappa, mu, matpc, dagger)
        assert_close(ref, P.to_host(out), prec, recon, f"tm_matpc matpc={matpc} dag={dagger}")
    # full operator through full fields
    full = P.spinor(seed=43, nparity=2)
    for dagger in (0, 1):
        out, inp = P.empty(2), P.to_dev(full, 2)
        D.ApplyTwistedMass(out, inp, P.U, -kappa, b_tw, inp, D.QUDA_INVALID_PARITY, dagger, backend=be)
        assert_close(oracle.tm_mat(P.gauge, full, X, kappa, mu, dagger), P.to_host(out), prec, recon, "tm_mat")


def check_multi_rhs(mem, be, prec, recon, n_src, op="wilson", xpay=False, dagger=0, X=(4, 6, 4, 8), nparity=1, comm_dim=None,
                    tile=None):
    """The reference's cvector_ref form: n_src sources sharing U (and A) in one call.  Every source is checked against
    the oracle AND must be bit-identical to its own single-source application (same arithmetic, same order)."""
    P = Problem(X, prec, recon, mem, clover=(op != "wilson"), compressed=True, dynamic=True)
    with_x = takes_x(op, xpay)
    a = -KAPPA if with_x else 0.0
    src = [P.spinor(seed=50 + i, nparity=nparity) for i in range(n_src)]
    xsrc = [P.spinor(seed=90 + i, nparity=nparity) for i in range(n_src)]
    parities = (0, 1) if nparity == 1 else (D.QUDA_INVALID_PARITY,)
    for parity in parities:
        ins = [P.to_dev(s, nparity) for s in src]
        xs = [P.to_dev(s, nparity) for s in xsrc] if with_x else None
        outs = [P.empty(nparity) for _ in range(n_src)]
        halo = None
        if comm_dim is not None:  # partitioned: the per-source fallback; one shared halo only makes sense for n_src == 1
            assert n_src == 1
            halo = self_halo(P, mem, comm_dim)
            self_exchange(P, halo, ins[0], 1 - parity, dagger, be)
        kw = dict(backend=be, tile=tile, halo=halo)
        apply(P, op, outs, ins, a, xs, parity, dagger, **kw)
        for i in range(n_src):
            one = P.empty(nparity)
            apply(P, op, one, ins[i], a, xs[i] if with_x else None, parity, dagger, **kw)
            got = P.to_host(outs[i])
            if nparity == 1:
                ref = reference(P, op, src[i], parity, dagger, xsrc[i] if with_x else None, a)
                assert_close(ref, got, prec, recon, f"multi-RHS {op} src {i}/{n_src} p={parity}")
            single = P.to_host(one)
            assert np.array_equal(got, single), \
                f"multi-RHS source {i} differs from its single-source application (max {np.abs(got - single).max():g})"


def self_halo(P, mem, comm_dim, nparity=1):
    """Ghost buffers for a single rank that is its own neighbour in every partitioned dimension."""
    h = D.Halo()
    for d in range(4):
        if comm_dim[d]:
            h.comm_dim[d] = 1
            for dir_ in range(2):
                h.ghost[d][dir_] = mem.empty(nparity * F.ghost_parity_bytes(P.X, P.prec, d))
    return h


def self_targets(halo):
    """Where a rank that is its own neighbour packs its faces, as PackGhost's dst[d][face]: our low face is what the
    backward neighbour receives from its forward side (ghost[d][1]); our high face is what the forward neighbour
    receives from its backward side (ghost[d][0])."""
    return [[halo.ghost[d][1], halo.ghost[d][0]] if halo.comm_dim[d] else [None, None] for d in range(4)]


def self_exchange(P, halo, in_field, in_parity, dagger, be, parity_slot=0):
    """PackGhost into our own receive buffers (self_targets), at the given parity slot of each buffer."""
    dst = [[None if buf is None else buf[parity_slot * F.ghost_parity_bytes(P.X, P.prec, d):] for buf in pair]
           for d, pair in enumerate(self_targets(halo))]
    D.PackGhost(dst, in_field, in_parity, dagger, halo.comm_dim, backend=be)


def check_partitioned(mem, be, prec, recon, comm_dim, op="wilson", X=(4, 4, 4, 4), xpay=False, dagger=0, clover_kw=None,
                      split=None, tile=None):
    """Self-partitioned run (the reference's --partition trick, tests/utils/host_utils.cpp:425): pack -> ghost buffers
    -> interior + fused exterior must reproduce the plain periodic operator.  `split` names the launches (SPLITS)."""
    P = Problem(X, prec, recon, mem, clover=(op != "wilson"), **(clover_kw or {}))
    s, xs = P.spinor(seed=31), P.spinor(seed=32)
    with_x = takes_x(op, xpay)
    a = -KAPPA if with_x else 0.0
    for parity in (0, 1):
        halo = self_halo(P, mem, comm_dim)
        din = P.to_dev(s)
        fused_kw = {}
        if split in ("fused", "fused_roles"):  # the launch packs the faces itself; host twin only: without arrival flags
            # the real kernel's boundary CTAs would not wait for its pack CTAs
            fused_kw = dict(fused_dst=self_targets(halo), block_counter=mem.empty(32))
        else:
            self_exchange(P, halo, din, 1 - parity, dagger, be)
        out = P.empty()
        xdev = P.to_dev(xs) if with_x else None
        for kw in SPLITS[split]:
            apply(P, op, out, din, a, xdev, parity, dagger, halo=halo, backend=be, tile=tile, **kw, **fused_kw)
        ref = reference(P, op, s, parity, dagger, xs if with_x else None, a)
        assert_close(ref, P.to_host(out), prec, recon, f"partitioned {comm_dim} op={op} p={parity}")


def check_partitioned_multi(mem, be, prec, recon, comm_dim, n_src, op="wilson", X=(4, 4, 4, 4), xpay=False, dagger=0,
                            clover_kw=None, split=None, aligned=True):
    """Batched halo of a multi-RHS batch on a self-partitioned lattice: ONE PackGhostMulti launch fills n_src ghost slabs
    per face, then every source's Dslash reads its own slab.  Each source must match the oracle AND be bit-identical to
    its own single-source partitioned application (same faces, same arithmetic)."""
    P = Problem(X, prec, recon, mem, clover=(op != "wilson"), **(clover_kw or {}))
    with_x = takes_x(op, xpay)
    a = -KAPPA if with_x else 0.0
    src = [P.spinor(seed=60 + i) for i in range(n_src)]
    xsrc = [P.spinor(seed=80 + i) for i in range(n_src)]
    face = [F.ghost_parity_bytes(P.X, prec, d) for d in range(4)]
    stride = [(fb + 255) // 256 * 256 if aligned else fb for fb in face]
    for parity in (0, 1):
        halo = D.Halo()
        halo.src_stride = stride
        for d in range(4):
            if comm_dim[d]:
                halo.comm_dim[d] = 1
                for dir_ in range(2):
                    halo.ghost[d][dir_] = mem.put(np.full(n_src * stride[d], 0x7B, dtype=np.uint8))  # poison: every slab must be written
        ins = [P.to_dev(s) for s in src]
        xs = [P.to_dev(s) for s in xsrc]
        D.PackGhostMulti(self_targets(halo), ins, 1 - parity, dagger, halo.comm_dim, stride, backend=be)

        def run(out, in_, x, h):
            for kw in SPLITS[split]:
                apply(P, op, out, in_, a, x if with_x else None, parity, dagger, halo=h, backend=be, **kw)

        # the whole batch in one call (b200_dslash_apply_multi: source i on slab i via halo.src_stride) ...
        outs = [P.empty() for _ in range(n_src)]
        run(outs, ins, xs, halo)
        for i in range(n_src):
            out = P.empty()
            run(out, ins[i], xs[i], halo.source(i))  # ... and source by source on the slab views
            got = P.to_host(out)
            assert np.array_equal(got, P.to_host(outs[i])), f"source {i}: batch call differs from the call on its slab view"
            ref = reference(P, op, src[i], parity, dagger, xsrc[i] if with_x else None, a)
            assert_close(ref, got, prec, recon, f"batched halo {comm_dim} op={op} src {i}/{n_src} p={parity}")
            single_halo = self_halo(P, mem, comm_dim)
            self_exchange(P, single_halo, ins[i], 1 - parity, dagger, be)
            one = P.empty()
            run(one, ins[i], xs[i], single_halo)
            assert np.array_equal(got, P.to_host(one)), f"source {i}: batched halo differs from its single-source exchange"
