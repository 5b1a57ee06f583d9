// Every host-side decision between the C ABI and a kernel launch that needs no CUDA: the entry points' validation,
// environment knobs and orchestration, the template dispatch, and the launch plans (which kernels, with which grids).
// The CUDA library (capi.cu, kernels.cuh, mrhs.cuh, tma_kernel.cuh) issues the plans with <<<>>>; the test-only host
// twin (tests/hosttwin) walks the same grids on the CPU, so the CPU test tier checks these decisions, not a copy of them.
#pragma once

#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <type_traits>

#include "launch.h"

#ifndef B2_MAXTILE
#define B2_MAXTILE 128
#endif
#ifndef B2_TMA_DEFAULT
#define B2_TMA_DEFAULT 0
#endif

namespace b200
{

  constexpr int kMaxTile = B2_MAXTILE; // threads per CTA of the tile kernels (kernels.cuh: occupancy targets)

  // ------------------------------------------------------------------ halo packing (kernels.cuh: pack_block)
  template <class P> struct PackArgs {
    Geom geom;
    SpinorView<P> in;
    GhostView<P> dst[4][2];
    unsigned *signal[4][2]; // remote arrival flags (nullptr: none)
    int *counter;           // 8 local block counters (zero between launches)
    unsigned seq;
    int comm_dim[4];
    int parity;
    int dagger;
  };

  // Which field a pack CTA reads and where its faces go: the launch's own (single exchange) ...
  template <class P> struct PackOwnViews {
    const PackArgs<P> &arg;
    B2_HD const SpinorView<P> &in() const { return arg.in; }
    B2_HD const GhostView<P> &dst(int d, int face) const { return arg.dst[d][face]; }
  };
  // ... or those of one source of a multi-RHS batch (pack_multi_kernel)
  template <class P> struct PackSourceViews {
    SpinorView<P> in_;
    GhostView<P> dst_;
    B2_HD const SpinorView<P> &in() const { return in_; }
    B2_HD const GhostView<P> &dst(int, int) const { return dst_; }
  };

  // the sources of a batched pack (pack_multi_kernel): source s reads in[s] and writes s * dst_stride[d] bytes behind the
  // first source's slab
  template <class P> struct PackBatch {
    typename P::store *in[B200_MAX_MULTI_RHS];
    float *in_norm[B200_MAX_MULTI_RHS];
    size_t dst_stride[4];
    int n_src;
  };

  // Face site `idx` of face `face` of dimension d: spin-project the boundary site and store the 12-real half spinor.
  // Face 0 (x[d] == 0) feeds the backward neighbour's forward hop, which uses P(d, dagger ? + : -);
  // face 1 (x[d] == X[d]-1) feeds the forward neighbour's backward hop, P(d, dagger ? - : +).
  // (reference: include/kernels/dslash_pack.cuh:134-200)
  template <class P, class Views> B2_HD void pack_site(const PackArgs<P> &arg, const Views &vw, int d, int face, int idx)
  {
    using real = typename P::real;
    const Geom &g = arg.geom;
    int x[4];
    coords_from_face(x, g, d, face ? g.X[d] - 1 : 0, idx, arg.parity);
    const int x_cb = cb_from_coords(x, g);
    const int sign = (face == 0) ? (arg.dagger ? +1 : -1) : (arg.dagger ? -1 : +1);
    real v[24], h[12];
    vw.in().load(v, x_cb);
    switch (d) {
    case 0: project(h, v, 0, sign); break;
    case 1: project(h, v, 1, sign); break;
    case 2: project(h, v, 2, sign); break;
    default: project(h, v, 3, sign); break;
    }
    vw.dst(d, face).save(h, idx);
  }

  template <class P> void fill_pack_args(PackArgs<P> &arg, const PackRequest &rq)
  {
    geom_init(arg.geom, rq.X);
    fill_spinor(arg.in, rq.in, rq.in_norm, arg.geom.volume_cb);
    arg.parity = rq.parity;
    arg.dagger = rq.dagger;
    arg.counter = rq.block_counter;
    arg.seq = rq.seq;
    for (int d = 0; d < 4; d++) {
      arg.comm_dim[d] = rq.comm_dim[d] ? 1 : 0;
      for (int dir = 0; dir < 2; dir++) {
        fill_ghost(arg.dst[d][dir], rq.dst[d][dir], rq.dst_norm[d][dir], arg.geom.face_cb[d]);
        arg.signal[d][dir] = arg.comm_dim[d] ? reinterpret_cast<unsigned *>(rq.signal[d][dir]) : nullptr;
      }
    }
  }

  template <class P> void fill_pack_batch(PackBatch<P> &batch, const PackBatchRequest &b, int volume_cb)
  {
    batch = PackBatch<P> {};
    batch.n_src = b.n_src;
    for (int s = 0; s < b.n_src; s++) {
      SpinorView<P> v;
      fill_spinor(v, b.in[s], b.in_norm[s], volume_cb);
      batch.in[s] = v.v;
      batch.in_norm[s] = v.norm;
    }
    for (int d = 0; d < 4; d++) batch.dst_stride[d] = b.dst_stride[d];
  }

  // grid.x of pack_kernel / pack_multi_kernel: CTAs of 128 threads over the largest partitioned face (0: nothing to pack)
  inline int pack_blocks(int &gx, const PackRequest &rq)
  {
    Geom g;
    geom_init(g, rq.X);
    int max_face = 0;
    bool any_signal = false;
    for (int d = 0; d < 4; d++) {
      if (!rq.comm_dim[d]) continue;
      if (g.face_cb[d] > max_face) max_face = g.face_cb[d];
      for (int dir = 0; dir < 2; dir++) any_signal |= (rq.signal[d][dir] != nullptr);
    }
    gx = (max_face + 127) / 128;
    if (gx && any_signal && !rq.block_counter) return set_error(B200_ERR_INVALID, "signal[] given without block_counter scratch");
    return 0;
  }

  // ------------------------------------------------------------------ ONE launch per partitioned Dslash
  // Block order of dslash_fused_kernel: [pack | interior part 1 | boundary | interior part 2]
  struct FusedShape {
    int n_pack, n_interior, n_boundary;
    int n_interior_first; // interior CTAs dispatched before the boundary CTAs (the rest follow them)
    int pack_start[9];    // prefix sums of the pack CTAs per face id
    int gx, gy;           // interior tile grid (gz implied)
  };

  // Block index decode of dslash_fused_kernel, for the host twin.  The kernel keeps its own inline copy (called as
  // these helpers, its machine code changes): change both together.
  // Block b < n_pack: a pack CTA of this face id
  inline int fused_pack_face(const FusedShape &fs, int b)
  {
    int f = 0;
    for (int k = 1; k < 8; k++)
      if (b >= fs.pack_start[k]) f = k;
    return f;
  }

  // Block n_pack + b: interior tile number ib >= 0 of the box, or -1 for boundary CTA b - n_interior_first.  The boundary
  // CTAs start when most of the interior is already in flight (by then the neighbours' faces have landed) and their
  // latency is covered by the rest of the interior instead of forming the tail of the launch.
  inline int fused_interior_tile(const FusedShape &fs, int b)
  {
    int ib = -1;
    if (b < fs.n_interior_first)
      ib = b;
    else if (b >= fs.n_interior_first + fs.n_boundary)
      ib = b - fs.n_boundary;
    return ib;
  }

  // interior tile ib -> block index (bx, by, bz) of the box grid
  inline void fused_tile_block(const FusedShape &fs, int ib, int &bx, int &by, int &bz)
  {
    const int per_z = fs.gx * fs.gy;
    bz = ib / per_z;
    const int r = ib - bz * per_z;
    by = r / fs.gx;
    bx = r - by * fs.gx;
  }

  // percent of the interior CTAs of a fused launch dispatched before its boundary CTAs (B200_FUSED_BOUNDARY_AT, read once)
  inline int fused_boundary_at()
  {
    static int boundary_at = -1;
    if (boundary_at < 0) {
      const char *e = getenv("B200_FUSED_BOUNDARY_AT");
      boundary_at = e ? atoi(e) : 70;
      if (boundary_at < 0 || boundary_at > 100) boundary_at = 100;
    }
    return boundary_at;
  }

  // ------------------------------------------------------------------ single-source Dslash launch plan
  enum LaunchKind {
    LAUNCH_INTERIOR, // dslash_interior_kernel over the box of `tm` (masked: the partitioned variant, part = true)
    LAUNCH_BOUNDARY, // dslash_boundary_kernel over the slabs of `st`
    LAUNCH_EXTERIOR, // dslash_exterior_kernel: one thread per face site
    LAUNCH_FUSED,    // dslash_fused_kernel with shape `fs` (the pack role packs rq.fused_pack)
  };

  struct LaunchStep {
    LaunchKind kind;
    bool masked;
    int grid[3], threads;
    TileMap tm;
    SlabTable st;
    FusedShape fs;
  };

  struct LaunchPlan {
    int n;
    LaunchStep step[2]; // issued in this order on rq.stream
    bool whole;         // the steps update every site of the operator
  };

  // OP_TM_PC_PRE (symmetric preconditioned twisted-mass dagger) is refused on a partitioned lattice (make_request), so
  // the executors build no masked-interior, boundary, exterior or fused step for it.
  constexpr bool has_partitioned_kernels(OpType op) { return op != OP_TM_PC_PRE; }

  // The launches of one Dslash request for the kernel arguments `arg` (DslashArgs of any precision / reconstruct)
  template <class Arg> int plan_dslash(LaunchPlan &pl, const LaunchRequest &rq, const Arg &arg)
  {
    pl.n = 0;
    pl.whole = false;
    TileMap tm {};
    int threads, gx, gy, gz, rc;
    if (int e = make_tile_map(tm, threads, rq.tile, arg.geom, kMaxTile)) return e;
    auto add = [&](LaunchKind kind, int x, int y, int thr) -> LaunchStep & {
      LaunchStep &l = pl.step[pl.n++];
      l.kind = kind;
      l.masked = false;
      l.grid[0] = x;
      l.grid[1] = y;
      l.grid[2] = 1;
      l.threads = thr;
      l.tm = tm;
      return l;
    };
    const int k = rq.kernel, n_parity = arg.n_parity;
    const bool partitioned = arg.threads_ext[4] > 0;
    const bool tiles_path = k == B200_KERNEL_AUTO || k == B200_KERNEL_INTERIOR_TILES || k == B200_KERNEL_BOUNDARY_TILES
      || k == B200_KERNEL_INTERIOR_SITES || k == B200_KERNEL_BOUNDARY_SITES;
    if (tiles_path && !partitioned && (k == B200_KERNEL_BOUNDARY_TILES || k == B200_KERNEL_BOUNDARY_SITES)) return 0;
    // the interior / boundary role of the fused kernel alone (1-site-thick shells, no pack role): what a caller with its
    // own pack launch puts on its main / side stream
    const bool sites = partitioned && n_parity == 1 && (k == B200_KERNEL_INTERIOR_SITES || k == B200_KERNEL_BOUNDARY_SITES);
    // roles of a fused launch: AUTO = pack | interior | boundary in one grid; INTERIOR_TILES = the interior role alone
    // (halo independent); BOUNDARY_TILES = pack | boundary (what a caller puts on a high-priority side stream)
    const bool fused = partitioned && rq.fused_pack && n_parity == 1
      && (k == B200_KERNEL_AUTO || k == B200_KERNEL_INTERIOR_TILES || k == B200_KERNEL_BOUNDARY_TILES);
    if (sites || fused) {
      if (fused && !rq.fused_pack->block_counter) return set_error(B200_ERR_INVALID, "fused Dslash needs the pack block_counter scratch");
      FusedShape fs {};
      const bool do_pack = fused && k != B200_KERNEL_INTERIOR_TILES;
      for (int f = 0; f < 8; f++) {
        const int d = f >> 1;
        const int nblk = (do_pack && rq.fused_pack->comm_dim[d]) ? (arg.geom.face_cb[d] + threads - 1) / threads : 0;
        fs.pack_start[f + 1] = fs.pack_start[f] + nblk;
      }
      fs.n_pack = fs.pack_start[8];
      if (!box_grid(tm, n_parity, gx, gy, gz, rc)) return rc ? rc : set_error(B200_ERR_INVALID, "empty lattice");
      fs.gx = gx;
      fs.gy = gy;
      fs.n_interior = (fused ? k != B200_KERNEL_BOUNDARY_TILES : k == B200_KERNEL_INTERIOR_SITES) ? gx * gy * gz : 0;
      fs.n_boundary = (fused ? k != B200_KERNEL_INTERIOR_TILES : k == B200_KERNEL_BOUNDARY_SITES) ? (arg.threads_ext[4] + threads - 1) / threads : 0;
      fs.n_interior_first = fused ? (int)((long long)fs.n_interior * fused_boundary_at() / 100) : fs.n_interior;
      add(LAUNCH_FUSED, fs.n_pack + fs.n_interior + fs.n_boundary, 1, threads).fs = fs;
      pl.whole = fused && k == B200_KERNEL_AUTO;
      return 0;
    }
    if (tiles_path && partitioned) {
      // Tile schedule: tiles that touch no partitioned face run now (branch-free kernel, overlapping the halo that is
      // in flight over NVLink); the boundary tiles follow in ONE launch that acquires the arrival flags and updates
      // its sites completely -- no partial sums, no read-modify-write pass.
      SlabTable st;
      const int nb = split_boundary(tm, st, arg.comm_dim);
      if (k != B200_KERNEL_BOUNDARY_TILES) {
        if (box_grid(tm, n_parity, gx, gy, gz, rc))
          add(LAUNCH_INTERIOR, gx, gy, threads).grid[2] = gz;
        else if (rc)
          return rc;
      }
      if (nb > 0 && k != B200_KERNEL_INTERIOR_TILES) add(LAUNCH_BOUNDARY, nb, n_parity, threads).st = st;
      pl.whole = k == B200_KERNEL_AUTO;
      return 0;
    }
    if (k != B200_KERNEL_EXTERIOR) { // AUTO / INTERIOR_TILES on an unpartitioned lattice, or reference-style INTERIOR
      if (!box_grid(tm, n_parity, gx, gy, gz, rc)) return rc ? rc : set_error(B200_ERR_INVALID, "empty lattice");
      LaunchStep &l = add(LAUNCH_INTERIOR, gx, gy, threads);
      l.grid[2] = gz;
      l.masked = partitioned;
      pl.whole = true;
    } else if (partitioned) {
      add(LAUNCH_EXTERIOR, (arg.threads_ext[4] + 127) / 128, n_parity, 128);
    }
    return 0;
  }

  // ------------------------------------------------------------------ multi-RHS launch grid (mrhs.cuh)
  struct MrhsGrid {
    TileMap tm;
    int threads, gx, gy, gz;
    int nsb, n_batch; // CTA flavour: sources per CTA, CTAs per tile
  };

  // grid of one multi-RHS launch over launch.h::mrhs_box (CTA flavour: `cta`); m.gx == 0: nothing to launch
  template <class Arg> int plan_mrhs(MrhsGrid &m, const MrhsRequest &rq, const Arg &arg, bool cta)
  {
    int rc;
    m.gx = 0;
    m.nsb = m.n_batch = 1;
    if (int e = make_tile_map(m.tm, m.threads, rq.base.tile, arg.geom, kMaxTile)) return e;
    if (!mrhs_box(m.tm, rq, arg.comm_dim, arg.n_parity, m.gx, m.gy, m.gz, rc)) {
      m.gx = 0;
      return rc;
    }
    if (cta) {
      mrhs_cta_shape(m.nsb, m.n_batch, rq.n_src, m.threads, kMaxTile, rq.cta_sources);
      if ((long long)m.gx * m.n_batch >= (1ll << 31)) return set_error(B200_ERR_INVALID, "lattice too large for the multi-RHS grid");
    }
    return 0;
  }

  // source `s` of a multi-RHS request as a single-source request
  inline LaunchRequest mrhs_source(const MrhsRequest &rq, int s)
  {
    LaunchRequest one = rq.base;
    one.out = rq.out[s];
    one.in = rq.in[s];
    if (rq.base.xpay) one.x = rq.x[s];
    return one;
  }

  // ------------------------------------------------------------------ template dispatch
  // compile-time configuration of one Dslash template instance (precision and reconstruct travel in DslashArgs<P, recon>)
  template <bool D, bool X, OpType O> struct OpCfg {
    static constexpr bool dagger = D, xpay = X;
    static constexpr OpType op = O;
  };

  // The op table: op x dagger x xpay -> template instance.  Fills the kernel arguments of the request's reconstruct and
  // calls f(OpCfg<dagger, xpay, op>{}, arg).
  template <class P, int recon, class F> int dispatch_op(const LaunchRequest &rq, F &f)
  {
    DslashArgs<P, recon> arg;
    if (int rc = fill_args(arg, rq)) return rc;
    const bool xp = rq.xpay, dg = rq.dagger;
    switch (rq.op) {
    case OP_WILSON:
      if (dg) return xp ? f(OpCfg<true, true, OP_WILSON> {}, arg) : f(OpCfg<true, false, OP_WILSON> {}, arg);
      return xp ? f(OpCfg<false, true, OP_WILSON> {}, arg) : f(OpCfg<false, false, OP_WILSON> {}, arg);
    case OP_CLOVER:
      if (!xp) return set_error(B200_ERR_INVALID, "ApplyWilsonClover exists in xpay form only (a != 0)");
      return dg ? f(OpCfg<true, true, OP_CLOVER> {}, arg) : f(OpCfg<false, true, OP_CLOVER> {}, arg);
    case OP_CLOVER_PC:
      if (dg) return xp ? f(OpCfg<true, true, OP_CLOVER_PC> {}, arg) : f(OpCfg<true, false, OP_CLOVER_PC> {}, arg);
      return xp ? f(OpCfg<false, true, OP_CLOVER_PC> {}, arg) : f(OpCfg<false, false, OP_CLOVER_PC> {}, arg);
    case OP_TM: // xpay form only
      return dg ? f(OpCfg<true, true, OP_TM> {}, arg) : f(OpCfg<false, true, OP_TM> {}, arg);
    case OP_TM_PC:
      if (dg && !rq.asymmetric) // symmetric dagger: the rotation acts on the neighbour spinors before the hop
        return xp ? f(OpCfg<true, true, OP_TM_PC_PRE> {}, arg) : f(OpCfg<true, false, OP_TM_PC_PRE> {}, arg);
      if (dg) return f(OpCfg<true, false, OP_TM_PC> {}, arg); // asymmetric dagger (never xpay)
      return xp ? f(OpCfg<false, true, OP_TM_PC> {}, arg) : f(OpCfg<false, false, OP_TM_PC> {}, arg);
    }
    return set_error(B200_ERR_INVALID, "unknown op %d", rq.op);
  }

  template <class P, class F> int dispatch_dslash(const LaunchRequest &rq, F &&f)
  {
    switch (rq.reconstruct) {
    case 18: return dispatch_op<P, 18>(rq, f);
    case 12: return dispatch_op<P, 12>(rq, f);
    case 8: return dispatch_op<P, 8>(rq, f);
    }
    return set_error(B200_ERR_INVALID, "reconstruct %d not in {18,12,8}", rq.reconstruct);
  }

  // The TMA-staged kernel serves unpartitioned fp64 / fp32 Wilson and clover requests (not clover-PC dagger with xpay);
  // anything else is kTmaSkip (the caller falls back to the gather kernels) and instantiates no TMA template.
  template <class P, class F> int dispatch_tma(const LaunchRequest &rq, F &&f)
  {
    return dispatch_dslash<P>(rq, [&](auto c, const auto &arg) -> int {
      using C = decltype(c);
      if constexpr (P::fixed || C::op == OP_TM || C::op == OP_TM_PC || C::op == OP_TM_PC_PRE || (C::op == OP_CLOVER_PC && C::dagger && C::xpay)) {
        return kTmaSkip;
      } else {
        if (arg.threads_ext[4] > 0) return kTmaSkip; // partitioned lattice: the halo schedule owns the launch
        return f(c, arg);
      }
    });
  }

  // TMA grid: one persistent CTA per SM (n_sm) unless B200_TMA_GRID says otherwise, never more CTAs than work items
  inline int tma_grid(const LaunchRequest &rq, int n_items, int n_sm)
  {
    const int grid = rq.tma_grid > 0 ? rq.tma_grid : n_sm;
    return grid > n_items ? n_items : grid;
  }

  // Multi-RHS ops (Wilson, clover, clover-PC): the CTA flavour (f(c, arg, 0, 0)), or batches of NS = 4 / 2 sources per
  // thread (f(c, arg, NS, s0)) with an odd source left over going through the single-source path (f(c, arg, 1, s0)).
  // NS travels as std::integral_constant.
  template <class P, class F> int dispatch_mrhs(const MrhsRequest &rq, F &&f)
  {
    return dispatch_dslash<P>(rq.base, [&](auto c, const auto &arg) -> int {
      if constexpr (decltype(c)::op > OP_CLOVER_PC) {
        return set_error(B200_ERR_INVALID, "unknown op %d", rq.base.op);
      } else {
        if (mrhs_mode(rq, P::bytes) == 1) return f(c, arg, std::integral_constant<int, 0> {}, 0);
        int s0 = 0;
        while (s0 < rq.n_src) {
          const int ns = mrhs_batch<P>(rq.n_src - s0, rq.max_batch);
          int rc;
          if (ns == 1)
            rc = f(c, arg, std::integral_constant<int, 1> {}, s0);
          else if (ns == 2)
            rc = f(c, arg, std::integral_constant<int, 2> {}, s0);
          else // fp64 never gets here (mrhs_batch caps it at 2) and instantiates no NS = 4 kernel
            rc = f(c, arg, std::integral_constant<int, P::bytes == 8 ? 2 : 4> {}, s0);
          if (rc) return rc;
          s0 += ns;
        }
        return B200_SUCCESS;
      }
    });
  }

  template <class F> int dispatch_precision(int precision, F &&f)
  {
    switch (precision) {
    case B200_DOUBLE: return f(PrecF64 {});
    case B200_SINGLE: return f(PrecF32 {});
    case B200_HALF: return f(PrecH16 {});
    }
    return set_error(B200_ERR_INVALID, "precision %d not in {8,4,2}", precision);
  }

  // ------------------------------------------------------------------ entry points
  // The bodies of the C entry points.  The executor E supplies require_device() and the per-precision launchers
  // dslash, tma (fp64 / fp32), mrhs, clover, twist, pack and pack_multi: the CUDA library (capi.cu) or the host twin.

  // B200_TMA=0|1|2 selects the TMA-staged marching kernel (2: fail instead of falling back when a shape is not served);
  // B200_TMA_TILE="ty tz", B200_TMA_GRID, B200_TMA_LINKS (n shared-memory stages, -1 register stream), B200_TMA_L2PF (L2
  // prefetch look-ahead in items, -1 off), B200_TMA_PREFETCH, B200_TMA_RINGS="centre halo" tune it.  Read on every call (a
  // handful of getenv lookups) so that tests and tuning scripts can switch between calls.
  inline void tma_knobs(LaunchRequest &rq)
  {
    const char *e = getenv("B200_TMA");
    rq.tma = e ? atoi(e) : B2_TMA_DEFAULT;
    if (!rq.tma) return;
    if ((e = getenv("B200_TMA_TILE"))) sscanf(e, "%d %d", &rq.tma_ty, &rq.tma_tz);
    if ((e = getenv("B200_TMA_GRID"))) rq.tma_grid = atoi(e);
    if ((e = getenv("B200_TMA_LINKS"))) rq.tma_link_slots = atoi(e);
    if ((e = getenv("B200_TMA_PREFETCH"))) rq.tma_prefetch = atoi(e);
    if ((e = getenv("B200_TMA_L2PF"))) rq.tma_l2_prefetch = atoi(e);
    if ((e = getenv("B200_TMA_RINGS"))) sscanf(e, "%d %d", &rq.tma_center_slots, &rq.tma_halo_slots);
  }

  template <class E> int apply_dslash(const b200_dslash_args *a)
  {
    if (int rc = E::require_device()) return rc;
    LaunchRequest rq;
    bool nothing_to_do = false;
    if (int rc = make_request(rq, a, nothing_to_do)) return rc;
    if (nothing_to_do) return B200_SUCCESS;
    tma_knobs(rq);
    if (rq.tma && rq.kernel == B200_KERNEL_AUTO && a->precision != B200_HALF) {
      // TMA-staged marching kernel (tma_kernel.cuh) for the shapes it serves; anything else falls through
      const int rc = a->precision == B200_DOUBLE ? E::template tma<PrecF64>(rq) : E::template tma<PrecF32>(rq);
      if (rc != kTmaSkip) return rc;
      if (rq.tma > 1) return set_error(B200_ERR_UNSUPPORTED, "B200_TMA=2: shape not served by the TMA kernel");
    }
    return dispatch_precision(a->precision, [&](auto p) { return E::template dslash<decltype(p)>(rq); });
  }

  template <class E>
  int apply_dslash_multi(const b200_dslash_args *a, int n_src, const b200_spinor *out, const b200_spinor *in, const b200_spinor *x)
  {
    if (int rc = E::require_device()) return rc;
    MrhsRequest rq;
    bool batched = false;
    if (int rc = make_mrhs_request(rq, a, n_src, out, in, x, batched)) return rc;
    if (!batched) { // other kernel selectors / operators: source by source, each on its own ghost slab
      for (int i = 0; i < n_src; i++) {
        const b200_dslash_args one = source_args(*a, i, out, in, x);
        if (int rc = apply_dslash<E>(&one)) return rc;
      }
      return B200_SUCCESS;
    }
    if (rq.interior_box && a->kernel == B200_KERNEL_AUTO) {
      // partitioned lattice, whole operator: the boundary tiles of every source (they wait for the batch's arrival counters
      // and read the source's own ghost slab) after the batched interior below -- the order the single-source AUTO path uses
      b200_dslash_args interior = *a;
      interior.kernel = B200_KERNEL_INTERIOR_TILES;
      if (int rc = apply_dslash_multi<E>(&interior, n_src, out, in, x)) return rc;
      for (int i = 0; i < n_src; i++) {
        b200_dslash_args one = source_args(*a, i, out, in, x);
        one.kernel = B200_KERNEL_BOUNDARY_TILES;
        if (int rc = apply_dslash<E>(&one)) return rc;
      }
      return B200_SUCCESS;
    }
    // tuning knobs (defaults are the measured best): B200_MRHS_MODE=thread|cta|auto, B200_MRHS_BATCH (sources per thread),
    // B200_MRHS_CTA_SOURCES (sources per CTA), B200_MRHS_L1=0|1 (link loads allocate in L1), B200_MRHS_CTA_CFG
    if (const char *e = getenv("B200_MRHS_MODE")) rq.mode = (strcmp(e, "cta") == 0) ? 1 : (strcmp(e, "thread") == 0 ? 0 : -1);
    if (const char *e = getenv("B200_MRHS_BATCH")) rq.max_batch = atoi(e);
    if (const char *e = getenv("B200_MRHS_CTA_SOURCES")) rq.cta_sources = atoi(e);
    if (const char *e = getenv("B200_MRHS_L1")) rq.l1_links = atoi(e) ? 1 : 0;
    if (const char *e = getenv("B200_MRHS_CTA_CFG")) rq.cta_cfg = atoi(e);
    return dispatch_precision(a->precision, [&](auto p) { return E::template mrhs<decltype(p)>(rq); });
  }

  inline int make_pack_request(PackRequest &rq, const b200_pack_args *a)
  {
    if (!a || !a->in.v) return set_error(B200_ERR_INVALID, "null argument");
    if (a->abi_version != B200_ABI_VERSION) return set_error(B200_ERR_INVALID, "ABI version mismatch");
    memcpy(rq.X, a->X, sizeof(rq.X));
    rq.parity = a->parity;
    rq.dagger = a->dagger ? 1 : 0;
    rq.in = a->in.v;
    rq.in_norm = a->in.norm;
    for (int d = 0; d < 4; d++) {
      rq.comm_dim[d] = a->comm_dim[d];
      for (int dir = 0; dir < 2; dir++) {
        rq.dst[d][dir] = a->dst[d][dir];
        rq.dst_norm[d][dir] = a->dst_norm[d][dir];
        rq.signal[d][dir] = a->signal[d][dir];
        if (a->comm_dim[d] && !a->dst[d][dir]) return set_error(B200_ERR_INVALID, "dst[%d][%d] is NULL", d, dir);
      }
    }
    rq.block_counter = a->block_counter;
    rq.seq = a->seq;
    rq.stream = a->stream;
    return 0;
  }

  template <class E> int apply_dslash_fused(const b200_dslash_args *a, const b200_pack_args *p)
  {
    if (int rc = E::require_device()) return rc;
    LaunchRequest rq;
    bool nothing_to_do = false;
    if (int rc = make_request(rq, a, nothing_to_do)) return rc;
    PackRequest pk;
    if (int rc = make_pack_request(pk, p)) return rc;
    if (a->kernel != B200_KERNEL_AUTO && a->kernel != B200_KERNEL_INTERIOR_TILES && a->kernel != B200_KERNEL_BOUNDARY_TILES)
      return set_error(B200_ERR_INVALID, "fused Dslash: kernel must be AUTO (all roles), INTERIOR_TILES (interior role) or BOUNDARY_TILES (pack + boundary roles)");
    if (p->in.v != a->in.v || p->precision != a->precision || p->parity != 1 - a->parity || (p->dagger != 0) != (a->dagger != 0))
      return set_error(B200_ERR_INVALID, "pack arguments do not describe the faces of this Dslash's input");
    if (a->out.n_parity != 1) return set_error(B200_ERR_INVALID, "the fused Dslash works on single-parity fields");
    bool any = false;
    for (int d = 0; d < 4; d++) {
      if ((p->comm_dim[d] != 0) != (a->halo.comm_dim[d] != 0)) return set_error(B200_ERR_INVALID, "pack / halo partitioning differ in dimension %d", d);
      if (p->X[d] != a->X[d]) return set_error(B200_ERR_INVALID, "pack / Dslash lattice extents differ");
      any |= a->halo.comm_dim[d] != 0;
    }
    if (!any) return a->kernel == B200_KERNEL_BOUNDARY_TILES ? B200_SUCCESS : apply_dslash<E>(a); // nothing partitioned: the plain launch
    if (a->halo.seq != p->seq) return set_error(B200_ERR_INVALID, "pack and halo carry different sequence numbers");
    rq.fused_pack = &pk;
    return dispatch_precision(a->precision, [&](auto p) { return E::template dslash<decltype(p)>(rq); });
  }

  template <class E> int pack_ghost(const b200_pack_args *a)
  {
    PackRequest rq;
    if (int rc = make_pack_request(rq, a)) return rc;
    if (int rc = E::require_device()) return rc;
    return dispatch_precision(a->precision, [&](auto p) { return E::template pack<decltype(p)>(rq); });
  }

  template <class E> int pack_ghost_multi(const b200_pack_args *a, int n_src, const b200_spinor *in, const size_t dst_stride[4])
  {
    if (n_src < 1 || n_src > B200_MAX_MULTI_RHS) return set_error(B200_ERR_INVALID, "n_src %d not in [1, %d]", n_src, B200_MAX_MULTI_RHS);
    if (!a || !in || !dst_stride) return set_error(B200_ERR_INVALID, "null argument");
    b200_pack_args first = *a;
    first.in = in[0];
    PackRequest rq;
    if (int rc = make_pack_request(rq, &first)) return rc;
    PackBatchRequest batch {};
    batch.n_src = n_src;
    for (int s = 0; s < n_src; s++) {
      if (!in[s].v) return set_error(B200_ERR_INVALID, "source %d is null", s);
      if (in[s].n_parity != 1) return set_error(B200_ERR_INVALID, "the batched pack takes single-parity sources");
      batch.in[s] = in[s].v;
      batch.in_norm[s] = in[s].norm;
    }
    for (int d = 0; d < 4; d++) batch.dst_stride[d] = dst_stride[d];
    if (int rc = check_src_stride("dst_stride", n_src, a->precision, a->X, a->comm_dim, dst_stride, 1)) return rc;
    if (int rc = E::require_device()) return rc;
    return dispatch_precision(a->precision, [&](auto p) { return E::template pack_multi<decltype(p)>(rq, batch); });
  }

  template <class E>
  int clover_apply(const b200_spinor *out, const b200_spinor *in, const b200_clover *A, int precision, int inverse, int parity, void *stream)
  {
    if (!out || !in || !A || !out->v || !in->v || !A->clover) return set_error(B200_ERR_INVALID, "null argument");
    if (int rc = E::require_device()) return rc;
    if (out->n_parity != 1 || in->n_parity != 1) return set_error(B200_ERR_INVALID, "ApplyClover acts on single-parity fields");
    if (parity != 0 && parity != 1) return set_error(B200_ERR_INVALID, "parity %d", parity);
    // inverse with a static-inverse build: the caller passes the A^-1 field and the kernel multiplies (same path as a
    // forward apply); with dynamic_inverse the field holds A and the kernel solves by Cholesky
    CloverRequest rq;
    rq.out = out->v;
    rq.out_norm = out->norm;
    rq.in = in->v;
    rq.in_norm = in->norm;
    rq.A = *A;
    rq.volume_cb = out->volume_cb;
    rq.inverse = inverse ? 1 : 0;
    rq.parity = parity;
    rq.stream = stream;
    return dispatch_precision(precision, [&](auto p) { return E::template clover<decltype(p)>(rq); });
  }

  // a, b of out = a (1 + i b gamma5) in for the singlet twist (dslash_gamma_helper.cuh:55-62)
  inline void twist_coefficients(double &a, double &b, double kappa, double mu, int dagger, int inverse)
  {
    if (!inverse) {
      b = 2.0 * kappa * mu;
      a = 1.0;
    } else {
      b = -2.0 * kappa * mu;
      a = 1.0 / (1.0 + b * b);
    }
    if (dagger) b = -b;
  }

  template <class E>
  int twist_gamma5(const b200_spinor *out, const b200_spinor *in, int precision, double kappa, double mu, int dagger, int inverse, void *stream)
  {
    if (!out || !in || !out->v || !in->v) return set_error(B200_ERR_INVALID, "b200_twist_gamma5: null argument");
    if (int rc = E::require_device()) return rc;
    if (out->n_parity != 1 || in->n_parity != 1 || out->volume_cb != in->volume_cb)
      return set_error(B200_ERR_INVALID, "b200_twist_gamma5 acts on single-parity fields of equal volume");
    TwistRequest rq;
    rq.out = out->v;
    rq.out_norm = out->norm;
    rq.in = in->v;
    rq.in_norm = in->norm;
    rq.volume_cb = out->volume_cb;
    twist_coefficients(rq.a, rq.b, kappa, mu, dagger, inverse);
    rq.stream = stream;
    return dispatch_precision(precision, [&](auto p) { return E::template twist<decltype(p)>(rq); });
  }

} // namespace b200
