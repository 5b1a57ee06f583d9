"""Operator-level parity cases shared by the CPU tier (host twin) and the GPU tier (libquda_b200.so)."""
import itertools

import numpy as np

import oracle
from common import Problem, assert_close
from quda_b200 import dslash as D
from quda_b200 import fields as F


def check_xpay_fullfield(mem, be, prec, recon, X=(4, 6, 4, 8)):
    P = Problem(X, prec, recon, mem, anisotropy=1.3)
    kappa = 0.12195
    s, xs = P.spinor(seed=3), P.spinor(seed=4)
    for parity, dagger in itertools.product((0, 1), (0, 1)):
        ref = xs.astype(np.float64) - kappa * oracle.wil_dslash(P.gauge, s, X, parity, dagger).astype(np.float64)
        out = P.empty()
        D.ApplyWilson(out, P.to_dev(s), P.U, -kappa, P.to_dev(xs), parity, dagger, backend=be)
        assert_close(ref, P.to_host(out), prec, recon, f"xpay p={parity} dag={dagger}")
    full = P.spinor(seed=9, nparity=2)
    for dagger in (0, 1):
        out, inp = P.empty(2), P.to_dev(full, 2)
        D.ApplyWilson(out, inp, P.U, -kappa, inp, D.QUDA_INVALID_PARITY, dagger, backend=be)
        assert_close(oracle.wil_mat(P.gauge, full, X, kappa, dagger), P.to_host(out), prec, recon, "full-field M")
        out2 = P.empty(2)
        D.ApplyWilson(out2, inp, P.U, 0.0, None, D.QUDA_INVALID_PARITY, dagger, backend=be)
        ref = np.concatenate([oracle.wil_dslash(P.gauge, full[P.Vh:], X, 0, dagger), oracle.wil_dslash(P.gauge, full[:P.Vh], X, 1, dagger)])
        assert_close(ref, P.to_host(out2), prec, recon, "full-field D")


def check_clover(mem, be, prec, recon, compressed, dynamic, X=(4, 4, 6, 4)):
    P = Problem(X, prec, recon, mem, clover=True, compressed=compressed, dynamic=dynamic)
    kappa = 0.12195
    s, xs = P.spinor(seed=21), P.spinor(seed=22)
    Ainv_field = P.A if dynamic else P.Ainv
    tolr = recon
    for parity in (0, 1):
        # ApplyClover: A x and A^{-1} x
        out = P.empty()
        D.ApplyClover(out, P.to_dev(s), P.A, False, parity, backend=be)
        assert_close(oracle.apply_clover(P.clover, s, X, parity), P.to_host(out), prec, tolr, "ApplyClover A")
        out = P.empty()
        D.ApplyClover(out, P.to_dev(s), Ainv_field, True, parity, backend=be)
        assert_close(oracle.apply_clover(P.clover_inv, s, X, parity), P.to_host(out), prec, tolr, "ApplyClover Ainv")
        for dagger in (0, 1):
            # preconditioned: A^{-1} D in
            out = P.empty()
            D.ApplyWilsonCloverPreconditioned(out, P.to_dev(s), P.U, Ainv_field, 0.0, None, parity, dagger, backend=be)
            ref = oracle.clover_dslash(P.gauge, P.clover_inv, s, X, parity, dagger)
            assert_close(ref, P.to_host(out), prec, tolr, f"clover-pc p={parity} dag={dagger}")
            # unpreconditioned xpay form: A x + a D in
            out = P.empty()
            D.ApplyWilsonClover(out, P.to_dev(s), P.U, P.A, -kappa, P.to_dev(xs), parity, dagger, backend=be)
            ref = oracle.apply_clover(P.clover, xs, X, parity).astype(np.float64) \
                - kappa * oracle.wil_dslash(P.gauge, s, X, parity, dagger).astype(np.float64)
            assert_close(ref, P.to_host(out), prec, tolr, f"clover xpay p={parity} dag={dagger}")
        # x + a A^{-1} D in (no dagger)
        out = P.empty()
        D.ApplyWilsonCloverPreconditioned(out, P.to_dev(s), P.U, Ainv_field, -kappa * kappa, P.to_dev(xs), parity, 0, backend=be)
        ref = xs.astype(np.float64) - kappa * kappa * oracle.clover_dslash(P.gauge, P.clover_inv, s, X, parity, 0).astype(np.float64)
        assert_close(ref, P.to_host(out), prec, tolr, "clover-pc xpay")


def check_twisted_mass(mem, be, prec, recon, X=(4, 6, 4, 8), comm_dim=None):
    """Degenerate twisted mass: ApplyTwistedMass / ApplyTwistedMassPreconditioned and their composition into the
    even-odd preconditioned operator for all four matpc types (lib/dirac_twisted_mass.cpp:47-237) against the oracle's
    tm_dslash / tm_mat / tm_matpc (tests/host_reference/wilson_dslash_reference.cpp:139-315)."""
    P = Problem(X, prec, recon, mem)
    kappa, mu = 0.12195, 0.1
    s, xs = P.spinor(seed=41), P.spinor(seed=42)
    f64 = np.float64
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
        D.ApplyTwistedMass(out, din, P.U, -kappa, b_tw, P.to_dev(xs), parity, dagger, halo=halo_for(din, 1 - parity, dagger),
                           backend=be)
        ref = oracle.twist_gamma5(xs, kappa, mu, dagger).astype(f64) - kappa * oracle.wil_dslash(P.gauge, s, X, parity, dagger).astype(f64)
        assert_close(ref, P.to_host(out), prec, recon, f"ApplyTwistedMass p={parity} dag={dagger}")
        # ApplyTwistedMassPreconditioned as DiracTwistedMassPC::Dslash / DslashXpay call it
        for matpc in range(4):
            asym = matpc >= 2 and dagger
            if comm_dim is not None and dagger and not asym:
                continue  # needs the twist in the pack kernel (rejected with B200_ERR_UNSUPPORTED, checked elsewhere)
            out = P.empty()
            D.ApplyTwistedMassPreconditioned(out, din, P.U, scale, a_inv, False, None, parity, dagger, asym,
                                             halo=halo_for(din, 1 - parity, dagger), backend=be)
            ref = oracle.tm_dslash(P.gauge, s, X, kappa, mu, parity, dagger, matpc).astype(f64)
            assert_close(ref, P.to_host(out), prec, recon, f"tm_dslash matpc={matpc} p={parity} dag={dagger}")
            if not asym:
                k = -kappa * kappa
                out = P.empty()
                D.ApplyTwistedMassPreconditioned(out, din, P.U, k * scale, a_inv, True, P.to_dev(xs), parity, dagger, False,
                                                 halo=halo_for(din, 1 - parity, dagger), backend=be)
                assert_close(xs.astype(f64) + k * ref, P.to_host(out), prec, recon, f"tm_dslash xpay matpc={matpc} dag={dagger}")
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
    kappa = 0.12195
    a = -kappa if xpay else 0.0
    src = [P.spinor(seed=50 + i, nparity=nparity) for i in range(n_src)]
    xsrc = [P.spinor(seed=90 + i, nparity=nparity) for i in range(n_src)]
    parities = (0, 1) if nparity == 1 else (D.QUDA_INVALID_PARITY,)
    for parity in parities:
        ins = [P.to_dev(s, nparity) for s in src]
        xs = [P.to_dev(s, nparity) for s in xsrc] if xpay else None
        outs = [P.empty(nparity) for _ in range(n_src)]
        halo = None
        if comm_dim is not None:  # partitioned: the per-source fallback; one shared halo only makes sense for n_src == 1
            assert n_src == 1
            halo = self_halo(P, mem, comm_dim)
            self_exchange(P, halo, ins[0], 1 - parity, dagger, be)
        kw = dict(backend=be, tile=tile, halo=halo)
        if op == "wilson":
            D.ApplyWilson(outs, ins, P.U, a, xs, parity, dagger, **kw)
        elif op == "clover_pc":
            D.ApplyWilsonCloverPreconditioned(outs, ins, P.U, P.A, a, xs, parity, dagger, **kw)
        else:
            D.ApplyWilsonClover(outs, ins, P.U, P.A, a, xs, parity, dagger, **kw)
        for i in range(n_src):
            one = P.empty(nparity)
            xi = xs[i] if xpay else None
            if op == "wilson":
                D.ApplyWilson(one, ins[i], P.U, a, xi, parity, dagger, **kw)
            elif op == "clover_pc":
                D.ApplyWilsonCloverPreconditioned(one, ins[i], P.U, P.A, a, xi, parity, dagger, **kw)
            else:
                D.ApplyWilsonClover(one, ins[i], P.U, P.A, a, xi, parity, dagger, **kw)
            got = P.to_host(outs[i])
            if nparity == 1:
                if op == "wilson":
                    ref = oracle.wil_dslash(P.gauge, src[i], X, parity, dagger).astype(np.float64)
                    if xpay:
                        ref = xsrc[i].astype(np.float64) - kappa * ref
                elif op == "clover_pc":
                    ref = oracle.clover_dslash(P.gauge, P.clover_inv, src[i], X, parity, dagger).astype(np.float64)
                    if xpay:
                        ref = xsrc[i].astype(np.float64) - kappa * ref
                else:
                    ref = oracle.apply_clover(P.clover, xsrc[i], X, parity).astype(np.float64) \
                        - kappa * oracle.wil_dslash(P.gauge, src[i], X, parity, dagger).astype(np.float64)
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


def self_exchange(P, halo, in_field, in_parity, dagger, be, parity_slot=0):
    """PackGhost into our own receive buffers: our low face is what the backward neighbour receives from its forward
    side (ghost[d][1]); our high face is what the forward neighbour receives from its backward side (ghost[d][0])."""
    dst = [[None, None] for _ in range(4)]
    for d in range(4):
        if halo.comm_dim[d]:
            off = parity_slot * F.ghost_parity_bytes(P.X, P.prec, d)
            dst[d][0] = halo.ghost[d][1][off:]
            dst[d][1] = halo.ghost[d][0][off:]
    D.PackGhost(dst, in_field, in_parity, dagger, halo.comm_dim, backend=be)


def check_partitioned(mem, be, prec, recon, comm_dim, op="wilson", X=(4, 4, 4, 4), xpay=False, dagger=0, clover_kw=None,
                      split=False, tile=None):
    """Self-partitioned run (the reference's --partition trick, tests/utils/host_utils.cpp:425): pack -> ghost buffers
    -> interior + fused exterior must reproduce the plain periodic operator."""
    P = Problem(X, prec, recon, mem, clover=(op != "wilson"), **(clover_kw or {}))
    kappa = 0.12195
    s, xs = P.spinor(seed=31), P.spinor(seed=32)
    for parity in (0, 1):
        halo = self_halo(P, mem, comm_dim)
        din = P.to_dev(s)
        fused_kw = {}
        if split in ("fused", "fused_roles"):  # pack + interior + boundary in one call (b200_dslash_apply_fused); host twin
            # only: without arrival flags the real kernel's boundary CTAs would not wait for its pack CTAs
            fused_kw = dict(fused_dst=[[halo.ghost[d][1], halo.ghost[d][0]] if comm_dim[d] else [None, None] for d in range(4)],
                            block_counter=mem.empty(32))
        else:
            self_exchange(P, halo, din, 1 - parity, dagger, be)
        out = P.empty()
        a = -kappa if xpay else 0.0
        xdev = P.to_dev(xs) if xpay else None
        if split == "tiles":      # the two halves of AUTO issued separately (boundary first: they are independent)
            kws = [dict(kernel=4, tile=tile), dict(kernel=3, tile=tile)]
        elif split == "sites":    # the same split with 1-site-thick shells (B200_KERNEL_BOUNDARY_SITES, then INTERIOR_SITES)
            kws = [dict(kernel=6, tile=tile), dict(kernel=5, tile=tile)]
        elif split == "fused_roles":  # the fused launch's roles as the `split` halo schedule issues them: pack + boundary
            # (B200_KERNEL_BOUNDARY_TILES), then the interior (B200_KERNEL_INTERIOR_TILES)
            kws = [dict(kernel=4, tile=tile, **fused_kw), dict(kernel=3, tile=tile, **fused_kw)]
        elif split and split != "fused":  # reference-style: masked INTERIOR then EXTERIOR read-modify-write
            kws = [dict(kernel=1, tile=tile), dict(kernel=2, tile=tile)]
        else:
            kws = [dict(tile=tile, **fused_kw)]
        if op == "wilson":
            for kw in kws:
                D.ApplyWilson(out, din, P.U, a, xdev, parity, dagger, halo=halo, backend=be, **kw)
            ref = oracle.wil_dslash(P.gauge, s, X, parity, dagger).astype(np.float64)
            if xpay:
                ref = xs.astype(np.float64) - kappa * ref
        elif op == "clover_pc":
            for kw in kws:
                D.ApplyWilsonCloverPreconditioned(out, din, P.U, P.A if P.A.dynamic else P.Ainv, a, xdev, parity, dagger,
                                                  halo=halo, backend=be, **kw)
            ref = oracle.clover_dslash(P.gauge, P.clover_inv, s, X, parity, dagger).astype(np.float64)
            if xpay:
                ref = xs.astype(np.float64) - kappa * ref
        else:
            for kw in kws:
                D.ApplyWilsonClover(out, din, P.U, P.A, -kappa, P.to_dev(xs), parity, dagger, halo=halo, backend=be, **kw)
            ref = oracle.apply_clover(P.clover, xs, X, parity).astype(np.float64) \
                - kappa * oracle.wil_dslash(P.gauge, s, X, parity, dagger).astype(np.float64)
        assert_close(ref, P.to_host(out), prec, recon, f"partitioned {comm_dim} op={op} p={parity}")


def check_partitioned_multi(mem, be, prec, recon, comm_dim, n_src, op="wilson", X=(4, 4, 4, 4), xpay=False, dagger=0,
                            clover_kw=None, split=None, aligned=True):
    """Batched halo of a multi-RHS batch on a self-partitioned lattice: ONE PackGhostMulti launch fills n_src ghost slabs
    per face, then every source's Dslash reads its own slab.  Each source must match the oracle AND be bit-identical to
    its own single-source partitioned application (same faces, same arithmetic)."""
    P = Problem(X, prec, recon, mem, clover=(op != "wilson"), **(clover_kw or {}))
    kappa = 0.12195
    a = -kappa if xpay or op == "clover" else 0.0
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
        dst = [[halo.ghost[d][1], halo.ghost[d][0]] if comm_dim[d] else [None, None] for d in range(4)]
        D.PackGhostMulti(dst, ins, 1 - parity, dagger, halo.comm_dim, stride, backend=be)
        if split == "tiles":
            kws = [dict(kernel=4), dict(kernel=3)]
        elif split == "sites":
            kws = [dict(kernel=6), dict(kernel=5)]
        else:
            kws = [dict()]

        def apply(out, i, h):
            xi = xs[i] if (xpay or op == "clover") else None
            for kw in kws:
                if op == "wilson":
                    D.ApplyWilson(out, ins[i], P.U, a, xi, parity, dagger, halo=h, backend=be, **kw)
                elif op == "clover_pc":
                    D.ApplyWilsonCloverPreconditioned(out, ins[i], P.U, P.A, a, xi, parity, dagger, halo=h, backend=be, **kw)
                else:
                    D.ApplyWilsonClover(out, ins[i], P.U, P.A, a, xi, parity, dagger, halo=h, backend=be, **kw)

        # the whole batch in one call (b200_dslash_apply_multi: source i on slab i via halo.src_stride) ...
        outs = [P.empty() for _ in range(n_src)]
        xl = xs if (xpay or op == "clover") else None
        for kw in kws:
            if op == "wilson":
                D.ApplyWilson(outs, ins, P.U, a, xl, parity, dagger, halo=halo, backend=be, **kw)
            elif op == "clover_pc":
                D.ApplyWilsonCloverPreconditioned(outs, ins, P.U, P.A, a, xl, parity, dagger, halo=halo, backend=be, **kw)
            else:
                D.ApplyWilsonClover(outs, ins, P.U, P.A, a, xl, parity, dagger, halo=halo, backend=be, **kw)
        for i in range(n_src):
            out = P.empty()
            apply(out, i, halo.source(i))  # ... and source by source on the slab views
            got = P.to_host(out)
            assert np.array_equal(got, P.to_host(outs[i])), f"source {i}: batch call differs from the call on its slab view"
            if op == "wilson":
                ref = oracle.wil_dslash(P.gauge, src[i], X, parity, dagger).astype(np.float64)
                if xpay:
                    ref = xsrc[i].astype(np.float64) - kappa * ref
            elif op == "clover_pc":
                ref = oracle.clover_dslash(P.gauge, P.clover_inv, src[i], X, parity, dagger).astype(np.float64)
                if xpay:
                    ref = xsrc[i].astype(np.float64) - kappa * ref
            else:
                ref = oracle.apply_clover(P.clover, xsrc[i], X, parity).astype(np.float64) \
                    - kappa * oracle.wil_dslash(P.gauge, src[i], X, parity, dagger).astype(np.float64)
            assert_close(ref, got, prec, recon, f"batched halo {comm_dim} op={op} src {i}/{n_src} p={parity}")
            single_halo = self_halo(P, mem, comm_dim)
            self_exchange(P, single_halo, ins[i], 1 - parity, dagger, be)
            one = P.empty()
            apply(one, i, single_halo)
            assert np.array_equal(got, P.to_host(one)), f"source {i}: batched halo differs from its single-source exchange"
