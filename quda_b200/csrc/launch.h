// Host-side glue between the precision-erased C ABI (include/b200_dslash.h) and the typed kernel arguments.
#pragma once

#include <cstdarg>
#include <cstdio>
#include <cuda_runtime.h>

#include "../../include/b200_dslash.h"
#include "dslash_site.h"

namespace b200
{

  int set_error(int code, const char *fmt, ...);
  int check_cuda(cudaError_t e, const char *what);
  void count_launch();

  struct LaunchRequest {
    int op, kernel, reconstruct, dagger, xpay, parity, n_parity;
    int X[4], tile[4];
    double b;       // twisted mass: twist factor as passed by the caller (the dagger sign flip happens in fill_args)
    int asymmetric; // twisted-mass preconditioned: asymmetric variant
    int tma;     // 1: unpartitioned single-source requests go to the TMA-staged marching kernel when it serves the shape
    int tma_ty, tma_tz, tma_grid; // tuning overrides of that kernel (0: built-in choice)
    int tma_link_slots;           // 0: links through shared memory, as many stages as fit; >= 2: that many; -1: register stream
    int tma_center_slots, tma_halo_slots; // cap the spinor rings (0: as deep as shared memory allows)
    int tma_l2_prefetch;          // shared-memory link stages: L2 prefetch look-ahead in items (0: built-in; < 0: off)
    int tma_prefetch;             // register-stream links: prefetch distance in direction pairs (2, 3 or 4; 0: built-in)
    double a;
    b200_spinor out, in, x;
    b200_gauge U;
    b200_clover A;
    b200_halo halo;
    void *stream;
    const struct PackRequest *fused_pack; // non-null: pack + interior + boundary in one launch (dslash_fused_kernel)
  };

  // multi-RHS: `base` carries everything but the spinors (its out/in/x mirror source 0 for validation)
  struct MrhsRequest {
    LaunchRequest base;
    int n_src;
    int max_batch; // sources per thread: 0 = built-in (4, fp64: 2); 1 disables in-thread batching
    int mode;      // 0: sources batched inside a thread (links in registers); 1: one thread per (site, source), sources
                   //    of a site in one CTA sharing the links through L1; -1: measured best per precision
                   //    and reconstruct (mrhs_mode below)
    int cta_sources; // mode 1: sources per CTA (0: as many as fit next to the tile in kMaxTile threads)
    int l1_links;  // mode 1: link loads allocate in L1 (1, default) or stream past it (0: repeats are served by L2)
    int cta_cfg;   // mode 1: occupancy configuration 0 / 1 / 2 (mrhs.cuh::MrhsCtaCfg)
    const b200_spinor *out, *in, *x;
    int interior_box; // partitioned lattice: only the tiles that touch no partitioned face (the boundary tiles follow per source)
  };

  struct CloverRequest {
    void *out, *out_norm, *in, *in_norm;
    b200_clover A;
    int volume_cb, inverse, parity;
    void *stream;
  };

  struct TwistRequest {
    void *out, *out_norm, *in, *in_norm;
    int volume_cb;
    double a, b; // out = a (in + b i gamma5 in)
    void *stream;
  };

  struct CopyRequest {
    void *native, *native_norm, *host;
    int volume_cb, host_precision, to_native;
    void *stream;
  };

  struct GaugeCopyRequest {
    b200_gauge native;
    int X[4];
    void *qdp[4], *ghost[4];
    int host_precision;
    void *stream;
  };

  struct CloverCopyRequest {
    b200_clover native;
    int X[4];
    const void *packed;
    int host_precision;
    void *stream;
  };

  struct PackRequest {
    int X[4], parity, dagger, comm_dim[4];
    void *in, *in_norm;
    void *dst[4][2], *dst_norm[4][2];
    void *signal[4][2];
    int *block_counter;
    unsigned seq;
    void *stream;
  };

  // bytes of one parity of one face buffer: 12 reals (+ a float norm in half precision) per checkerboard face site
  inline size_t ghost_parity_bytes(int precision, const int X[4], int dim)
  {
    const size_t face_cb = (size_t)X[0] * X[1] * X[2] * X[3] / X[dim] / 2;
    return face_cb * (12 * (size_t)precision + (precision == B200_HALF ? 4 : 0));
  }

  // ghost slabs of a multi-RHS batch: one per source, `stride[d]` bytes apart -- at least one slab, and 16-byte multiples so
  // that every slab keeps the alignment of the vector loads / stores
  inline int check_src_stride(const char *what, int n_src, int precision, const int X[4], const int comm_dim[4], const size_t stride[4],
                              int n_parity)
  {
    for (int d = 0; d < 4; d++) {
      if (!comm_dim[d] || n_src <= 1) continue;
      const size_t slab = (size_t)n_parity * ghost_parity_bytes(precision, X, d);
      if (stride[d] < slab)
        return set_error(B200_ERR_INVALID, "%s[%d] = %zu is smaller than one face (%zu bytes): every source needs its own ghost slab", what, d,
                         stride[d], slab);
      if (stride[d] % 16) return set_error(B200_ERR_INVALID, "%s[%d] = %zu is not a multiple of 16 bytes", what, d, stride[d]);
    }
    return 0;
  }

  // A batch of sources packed by ONE launch (b200_pack_ghost_multi): source s reads in[s] and writes its faces
  // dst_stride[d] * s bytes behind the first source's slab in dimension d; the arrival counters move once, for all of them.
  struct PackBatchRequest {
    int n_src;
    void *in[B200_MAX_MULTI_RHS], *in_norm[B200_MAX_MULTI_RHS];
    size_t dst_stride[4];
  };

  template <class P> void fill_spinor(SpinorView<P> &v, void *base, void *norm, int volume_cb)
  {
    v.v = reinterpret_cast<typename P::store *>(base);
    v.stride = volume_cb;
    if (P::fixed)
      v.norm = norm ? reinterpret_cast<float *>(norm) :
                      reinterpret_cast<float *>(reinterpret_cast<short *>(base) + (size_t)24 * volume_cb);
    else
      v.norm = nullptr;
  }

  // parity block `p` of a b200_spinor
  template <class P> void fill_spinor_parity(SpinorView<P> &v, const b200_spinor &f, int p)
  {
    char *base = reinterpret_cast<char *>(f.v) + (size_t)p * f.parity_stride_bytes;
    char *norm = f.norm ? reinterpret_cast<char *>(f.norm) + (size_t)p * f.parity_stride_bytes : nullptr;
    fill_spinor(v, base, norm, f.volume_cb);
  }

  template <class P> void fill_clover(CloverView<P> &A, const b200_clover &c, int volume_cb)
  {
    A.c[0] = reinterpret_cast<const typename P::store *>(c.clover);
    A.c[1] = reinterpret_cast<const typename P::store *>(reinterpret_cast<const char *>(c.clover) + c.parity_stride_bytes);
    A.volume_cb = volume_cb;
    A.compressed = c.compressed;
    A.dynamic = c.dynamic_inverse;
    A.diagonal = (typename P::real)c.diagonal;
    A.nrm = (float)(c.max_element / (2.0 * 32767.0)); // clover_field_order.h:621-624
  }

  template <class P> void fill_ghost(GhostView<P> &g, void *base, void *norm, int face_cb)
  {
    g.v = reinterpret_cast<typename P::store *>(base);
    g.face_cb = face_cb;
    if (P::fixed)
      g.norm = norm ? reinterpret_cast<float *>(norm) :
                      (base ? reinterpret_cast<float *>(reinterpret_cast<short *>(base) + (size_t)12 * face_cb) : nullptr);
    else
      g.norm = nullptr;
  }

  // ghost slab of source `s` in a batched exchange: `bytes` = s * (the caller's slab stride in this dimension)
  template <class P> B2_HD GhostView<P> ghost_of_source(GhostView<P> g, size_t bytes)
  {
    g.v = reinterpret_cast<typename P::store *>(reinterpret_cast<char *>(g.v) + bytes);
    if (g.norm) g.norm = reinterpret_cast<float *>(reinterpret_cast<char *>(g.norm) + bytes);
    return g;
  }

  template <class P, int recon> int fill_args(DslashArgs<P, recon> &arg, const LaunchRequest &rq)
  {
    geom_init(arg.geom, rq.X);
    const Geom &g = arg.geom;
    arg.n_parity = rq.n_parity;
    arg.parity = rq.parity;
    arg.a = (typename P::real)rq.a;
    arg.A = CloverView<P> {};
    arg.A.diagonal = (typename P::real)(rq.dagger ? -rq.b : rq.b); // twist_b(); dslash_twisted_mass.cuh:27: "if dagger flip the twist"
    if (rq.out.volume_cb != g.volume_cb || rq.in.volume_cb != g.volume_cb)
      return set_error(B200_ERR_INVALID, "spinor volume_cb (%d/%d) does not match lattice (%d)", rq.out.volume_cb,
                       rq.in.volume_cb, g.volume_cb);
    if (rq.n_parity == 2) {
      for (int p = 0; p < 2; p++) {
        fill_spinor_parity(arg.out[p], rq.out, p);
        fill_spinor_parity(arg.in[p], rq.in, p);
        if (rq.xpay) fill_spinor_parity(arg.x[p], rq.x, p);
      }
    } else { // single-parity fields: `out`/`x` hold parity `parity`, `in` holds the other one
      fill_spinor_parity(arg.out[rq.parity], rq.out, 0);
      fill_spinor_parity(arg.in[1 - rq.parity], rq.in, 0);
      if (rq.xpay) fill_spinor_parity(arg.x[rq.parity], rq.x, 0);
    }
    GaugeMeta m;
    m.anisotropy = rq.U.anisotropy;
    m.link_max = rq.U.link_max;
    m.t_boundary = rq.U.t_boundary;
    m.first_time_slice = rq.U.first_time_slice;
    m.last_time_slice = rq.U.last_time_slice;
    m.t_bound_cb = (g.X[3] - 1) * g.X[0] * g.X[1] * g.X[2] / 2;
    m.volume_cb = g.volume_cb;
    arg.U.init(rq.U.gauge, rq.U.parity_stride_bytes, rq.U.stride, m);
    if (rq.op == OP_CLOVER || rq.op == OP_CLOVER_PC) fill_clover(arg.A, rq.A, g.volume_cb);
    arg.threads_ext[0] = 0;
    for (int d = 0; d < 4; d++) {
      arg.comm_dim[d] = rq.halo.comm_dim[d] ? 1 : 0;
      if (arg.comm_dim[d] && g.X[d] < 4)
        return set_error(B200_ERR_INVALID, "partitioned dimension %d needs local extent >= 4 (got %d)", d, g.X[d]);
      arg.threads_ext[d + 1] = arg.threads_ext[d] + (arg.comm_dim[d] ? 2 * g.face_cb[d] : 0);
      const size_t parity_elems = (size_t)12 * g.face_cb[d] + (P::fixed ? 2 * g.face_cb[d] : 0); // norms: 1 float = 2 shorts
      arg.ghost_parity_stride[d] = rq.n_parity == 2 ? parity_elems : 0;
      arg.ghost_norm_parity_stride[d] = rq.n_parity == 2 ? parity_elems / 2 : 0;
      for (int dir = 0; dir < 2; dir++) {
        if (arg.comm_dim[d] && rq.kernel != B200_KERNEL_INTERIOR && rq.kernel != B200_KERNEL_INTERIOR_TILES
            && rq.kernel != B200_KERNEL_INTERIOR_SITES && !rq.halo.ghost[d][dir])
          return set_error(B200_ERR_INVALID, "dimension %d is partitioned but halo.ghost[%d][%d] is NULL", d, d, dir);
        fill_ghost(arg.ghost[d][dir], rq.halo.ghost[d][dir], rq.halo.ghost_norm[d][dir], g.face_cb[d]);
        arg.wait_flag[d][dir] = arg.comm_dim[d] ? reinterpret_cast<const unsigned *>(rq.halo.wait_flag[d][dir]) : nullptr;
      }
    }
    arg.seq = rq.halo.seq;
    arg.timeout_flag = rq.halo.timeout_flag;
    return 0;
  }


  // sources handled by one thread in the next multi-RHS launch: as many as the register file carries
  // (fp32 / half: 4, fp64: 2), then 2, then the single-source kernel
  template <class P> int mrhs_batch(int remaining, int max_batch)
  {
    int cap = sizeof(typename P::real) == 8 ? 2 : 4;
    if (max_batch > 0 && max_batch < cap) cap = max_batch;
    if (remaining >= 4 && cap >= 4) return 4;
    if (remaining >= 2 && cap >= 2) return 2;
    return 1;
  }

  template <class P, int NS> void fill_mrhs_fields(MrhsFields<P, NS> &f, const MrhsRequest &rq, int s0)
  {
    const LaunchRequest &b = rq.base;
    for (int s = 0; s < NS; s++) {
      for (int p = 0; p < 2; p++) {
        f.out[s][p] = SpinorView<P> {};
        f.in[s][p] = SpinorView<P> {};
        f.x[s][p] = SpinorView<P> {};
      }
      if (b.n_parity == 2) {
        for (int p = 0; p < 2; p++) {
          fill_spinor_parity(f.out[s][p], rq.out[s0 + s], p);
          fill_spinor_parity(f.in[s][p], rq.in[s0 + s], p);
          if (b.xpay) fill_spinor_parity(f.x[s][p], rq.x[s0 + s], p);
        }
      } else {
        fill_spinor_parity(f.out[s][b.parity], rq.out[s0 + s], 0);
        fill_spinor_parity(f.in[s][1 - b.parity], rq.in[s0 + s], 0);
        if (b.xpay) fill_spinor_parity(f.x[s][b.parity], rq.x[s0 + s], 0);
      }
    }
  }

  template <class P> void fill_mrhs_views(MrhsViews<P> &f, const MrhsRequest &rq)
  {
    static_assert(kMaxRhs == B200_MAX_MULTI_RHS, "kMaxRhs mirrors the C ABI limit");
    const LaunchRequest &b = rq.base;
    for (int s = 0; s < kMaxRhs; s++)
      for (int p = 0; p < 2; p++) {
        f.out[s][p] = SpinorView<P> {};
        f.in[s][p] = SpinorView<P> {};
        f.x[s][p] = SpinorView<P> {};
      }
    for (int s = 0; s < rq.n_src; s++) {
      if (b.n_parity == 2) {
        for (int p = 0; p < 2; p++) {
          fill_spinor_parity(f.out[s][p], rq.out[s], p);
          fill_spinor_parity(f.in[s][p], rq.in[s], p);
          if (b.xpay) fill_spinor_parity(f.x[s][p], rq.x[s], p);
        }
      } else {
        fill_spinor_parity(f.out[s][b.parity], rq.out[s], 0);
        fill_spinor_parity(f.in[s][1 - b.parity], rq.in[s], 0);
        if (b.xpay) fill_spinor_parity(f.x[s][b.parity], rq.x[s], 0);
      }
    }
  }

  inline int mrhs_mode(const MrhsRequest &rq, int precision)
  {
    if (rq.mode == 0 || rq.mode == 1) return rq.mode;
    // the CTA flavour shares each tile's links between the sources of a CTA; it pays where the links are a large share
    // of the traffic (fp64, fp32 recon-12)
    if (precision == B200_DOUBLE) return 1;
    if (precision == B200_SINGLE && rq.base.reconstruct == 12) return 1;
    return 0;
  }

  // CTA flavour launch shape: `tile_threads` sites x `nsb` sources per CTA (<= max_threads), n_batch CTAs per tile
  inline void mrhs_cta_shape(int &nsb, int &n_batch, int n_src, int tile_threads, int max_threads, int requested)
  {
    nsb = max_threads / tile_threads;
    if (nsb < 1) nsb = 1;
    if (requested > 0 && requested < nsb) nsb = requested;
    if (nsb > n_src) nsb = n_src;
    n_batch = (n_src + nsb - 1) / nsb;
  }

  // default launch geometry per precision: tile of checkerboard sites (x/2, y, z, t), see DESIGN.md
  inline void default_tile(int *tile, int precision, const int *X)
  {
    // full x rows (coalesced 256..512-byte runs per plane) and small CTAs (bench.py --sweep times the alternatives)
    int t[4] = {16, 2, 2, 1};
    if (precision == B200_DOUBLE) { t[0] = 16; t[1] = 2; t[2] = 1; t[3] = 1; }
    if (precision == B200_HALF) { t[0] = 16; t[1] = 8; t[2] = 1; t[3] = 1; }
    for (int d = 0; d < 4; d++) {
      const int ext = d == 0 ? X[0] / 2 : X[d];
      while (t[d] > 1 && ext % t[d] != 0) t[d] /= 2;
      if (t[d] > ext) t[d] = ext;
      tile[d] = t[d];
    }
  }

  // The symmetric preconditioned twisted-mass dagger rotates the neighbour spinors before the hop.  The pack kernel does
  // not rotate the faces it sends, so this op is refused on a partitioned lattice and has no partitioned kernels
  // (plan.h::has_partitioned_kernels).
  inline int refuse_partitioned_tm_pc_pre()
  {
    return set_error(B200_ERR_UNSUPPORTED, "symmetric preconditioned twisted-mass dagger on a partitioned lattice needs the "
                                           "twist in the pack kernel: not built");
  }

  // Validate a b200_dslash_args block and turn it into the precision-erased launch request
  // (shared by the CUDA library and the test-only host twin so both see identical argument semantics).
  inline int make_request(LaunchRequest &rq, const b200_dslash_args *a, bool &nothing_to_do)
  {
    nothing_to_do = false;
    if (!a) return set_error(B200_ERR_INVALID, "null args");
    if (a->abi_version != B200_ABI_VERSION)
      return set_error(B200_ERR_INVALID, "ABI version mismatch: caller %d, library %d", a->abi_version, B200_ABI_VERSION);
    for (int d = 0; d < 4; d++)
      if (a->X[d] < 2 || (a->X[d] & 1)) return set_error(B200_ERR_INVALID, "X[%d]=%d must be even and >= 2", d, a->X[d]);
    if (!a->out.v || !a->in.v || !a->U.gauge) return set_error(B200_ERR_INVALID, "null field pointer");
    if (a->out.v == a->in.v) return set_error(B200_ERR_INVALID, "out and in must not alias (dslash_helper.cuh:355)");
    if (a->out.n_parity != a->in.n_parity || (a->out.n_parity != 1 && a->out.n_parity != 2))
      return set_error(B200_ERR_INVALID, "out/in site subsets differ or are invalid (%d/%d)", a->out.n_parity, a->in.n_parity);
    if (a->out.n_parity == 1 && a->parity != 0 && a->parity != 1)
      return set_error(B200_ERR_INVALID, "parity %d invalid for single-parity fields", a->parity);
    if (a->op < B200_OP_WILSON || a->op > B200_OP_TWISTED_MASS_PC) return set_error(B200_ERR_INVALID, "unknown op %d", a->op);
    const bool clover_op = a->op == B200_OP_CLOVER || a->op == B200_OP_CLOVER_PC;
    if (clover_op && !a->A.clover) return set_error(B200_ERR_INVALID, "clover operator without clover field");
    bool any_comm_tm = false;
    for (int d = 0; d < 4; d++) any_comm_tm |= (a->halo.comm_dim[d] != 0);
    if (a->op == B200_OP_TWISTED_MASS && a->a == 0.0)
      return set_error(B200_ERR_INVALID, "Twisted-mass operator only defined for xpay=true (a != 0)"); // lib/dslash_twisted_mass.cu
    if (a->op == B200_OP_TWISTED_MASS_PC) { // lib/dslash_twisted_mass_preconditioned.cu:41-43
      if (a->asymmetric && !a->dagger) return set_error(B200_ERR_INVALID, "asymmetric operator only defined for dagger");
      if (a->asymmetric && a->x.v) return set_error(B200_ERR_INVALID, "asymmetric operator not defined for xpay");
      if (a->out.n_parity != 1) return set_error(B200_ERR_INVALID, "Preconditioned twisted-mass operator not defined nParity=2");
      if (a->dagger && !a->asymmetric && any_comm_tm) return refuse_partitioned_tm_pc_pre();
    }
    if (a->op == B200_OP_CLOVER_PC && a->out.n_parity != 1)
      return set_error(B200_ERR_INVALID, "preconditioned clover operator only defined on single-parity fields");
    if (a->op == B200_OP_CLOVER_PC && a->a != 0.0 && a->dagger)
      return set_error(B200_ERR_INVALID, "xpay with dagger is not defined for the preconditioned clover operator");
    if (a->precision != B200_DOUBLE && a->precision != B200_SINGLE && a->precision != B200_HALF)
      return set_error(B200_ERR_INVALID, "precision %d not in {8,4,2}", a->precision);
    rq.op = a->op;
    rq.kernel = a->kernel;
    rq.reconstruct = a->U.reconstruct;
    rq.dagger = a->dagger ? 1 : 0;
    rq.xpay = (a->op == B200_OP_TWISTED_MASS_PC) ? (a->x.v != nullptr) : (a->a != 0.0);
    rq.a = a->a;
    rq.b = a->b;
    rq.asymmetric = a->asymmetric ? 1 : 0;
    rq.parity = a->parity;
    rq.n_parity = a->out.n_parity;
    for (int d = 0; d < 4; d++) rq.X[d] = a->X[d];
    if (a->tile[0] > 0) {
      for (int d = 0; d < 4; d++) rq.tile[d] = a->tile[d] > 0 ? a->tile[d] : 1;
    } else {
      default_tile(rq.tile, a->precision, a->X);
    }
    rq.fused_pack = nullptr;
    rq.tma = 0;
    rq.tma_ty = rq.tma_tz = rq.tma_grid = rq.tma_link_slots = rq.tma_center_slots = rq.tma_halo_slots = rq.tma_prefetch = rq.tma_l2_prefetch = 0;
    rq.out = a->out;
    rq.in = a->in;
    rq.x = a->x;
    if (rq.xpay && !rq.x.v) return set_error(B200_ERR_INVALID, "a != 0 but x is null");
    rq.U = a->U;
    rq.A = a->A;
    rq.halo = a->halo;
    rq.stream = a->stream;
    bool any_comm = false;
    for (int d = 0; d < 4; d++) any_comm |= (a->halo.comm_dim[d] != 0);
    if (rq.kernel < B200_KERNEL_AUTO || rq.kernel > B200_KERNEL_BOUNDARY_SITES)
      return set_error(B200_ERR_INVALID, "unknown kernel selector %d", rq.kernel);
    if ((rq.kernel == B200_KERNEL_EXTERIOR || rq.kernel == B200_KERNEL_BOUNDARY_TILES || rq.kernel == B200_KERNEL_BOUNDARY_SITES) && !any_comm)
      nothing_to_do = true;
    return 0;
  }

  // Validate the multi-RHS form: `a` as for b200_dslash_apply (its out/in/x are ignored), n_src sources sharing U / A.
  // `batched` comes back false when the request must run source by source (partitioned lattice or an explicit
  // kernel selector: the halo schedule is per source).
  inline int make_mrhs_request(MrhsRequest &rq, const b200_dslash_args *a, int n_src, const b200_spinor *out,
                               const b200_spinor *in, const b200_spinor *x, bool &batched)
  {
    if (!a) return set_error(B200_ERR_INVALID, "null args");
    if (n_src < 1 || n_src > B200_MAX_MULTI_RHS)
      return set_error(B200_ERR_INVALID, "n_src %d not in [1, %d]", n_src, B200_MAX_MULTI_RHS);
    if (!out || !in) return set_error(B200_ERR_INVALID, "null source / destination array");
    if (a->a != 0.0 && !x) return set_error(B200_ERR_INVALID, "a != 0 but x is null");
    for (int i = 0; i < n_src; i++) {
      if (out[i].n_parity != out[0].n_parity || in[i].n_parity != out[0].n_parity || out[i].volume_cb != out[0].volume_cb
          || in[i].volume_cb != out[0].volume_cb)
        return set_error(B200_ERR_INVALID, "source %d: site subset / volume differs from source 0", i);
      if (!out[i].v || !in[i].v || (a->a != 0.0 && !x[i].v)) return set_error(B200_ERR_INVALID, "source %d: null field pointer", i);
      for (int j = 0; j < n_src; j++) {
        if (out[i].v == in[j].v) return set_error(B200_ERR_INVALID, "out[%d] aliases in[%d]", i, j);
        if (j != i && out[i].v == out[j].v) return set_error(B200_ERR_INVALID, "out[%d] aliases out[%d]", i, j);
      }
    }
    b200_dslash_args first = *a;
    first.out = out[0];
    first.in = in[0];
    if (a->a != 0.0) first.x = x[0];
    bool nothing = false;
    if (int rc = make_request(rq.base, &first, nothing)) return rc;
    rq.n_src = n_src;
    rq.max_batch = 0;
    rq.mode = -1;
    rq.cta_sources = 0;
    rq.l1_links = 1;
    rq.cta_cfg = 0;
    rq.out = out;
    rq.in = in;
    rq.x = x;
    bool any_comm = false;
    for (int d = 0; d < 4; d++) any_comm |= (a->halo.comm_dim[d] != 0);
    // every source needs its own ghost slab (one b200_pack_ghost_multi fills them all)
    if (int rc = check_src_stride("halo.src_stride", n_src, a->precision, a->X, a->halo.comm_dim, a->halo.src_stride, out[0].n_parity)) return rc;
    // batched kernels serve whole unpartitioned lattices and, on partitioned ones, the interior tiles (no ghost zones there:
    // the same branch-free site code); boundary tiles / other kernel selectors run source by source
    // (a single source on a partitioned lattice gains nothing from that and keeps the plain single-source path)
    rq.interior_box = any_comm ? 1 : 0;
    batched = a->op <= B200_OP_CLOVER_PC
      && (any_comm ? n_src > 1 && (a->kernel == B200_KERNEL_AUTO || a->kernel == B200_KERNEL_INTERIOR_TILES) : a->kernel == B200_KERNEL_AUTO);
    return 0;
  }

  // source `i` of a multi-RHS batch as a single-source call: its own fields and, on a partitioned lattice, its own ghost slab
  inline b200_dslash_args source_args(const b200_dslash_args &a, int i, const b200_spinor *out, const b200_spinor *in, const b200_spinor *x)
  {
    b200_dslash_args one = a;
    one.out = out[i];
    one.in = in[i];
    if (a.a != 0.0) one.x = x[i];
    for (int d = 0; d < 4; d++)
      for (int dir = 0; dir < 2; dir++) {
        const size_t off = (size_t)i * a.halo.src_stride[d];
        if (one.halo.ghost[d][dir]) one.halo.ghost[d][dir] = static_cast<char *>(a.halo.ghost[d][dir]) + off;
        if (one.halo.ghost_norm[d][dir]) one.halo.ghost_norm[d][dir] = static_cast<char *>(a.halo.ghost_norm[d][dir]) + off;
      }
    return one;
  }

  // launch geometry of the interior kernel for a requested tile (extents rounded down to powers of two); the box
  // initially covers all tiles
  inline int make_tile_map(TileMap &tm, int &threads, const int *tile, const Geom &g, int max_threads)
  {
    threads = 1;
    for (int d = 0; d < 4; d++) {
      int sh = 0;
      while ((2 << sh) <= tile[d]) sh++;
      const int ext = d == 0 ? g.Xh0 : g.X[d];
      while (sh > 0 && (1 << sh) > 2 * ext) sh--; // no point in tiles more than twice the extent
      tm.sh[d] = sh;
      tm.nt[d] = (ext + (1 << sh) - 1) >> sh;
      tm.org[d] = 0;
      tm.cnt[d] = tm.nt[d];
      threads <<= sh;
    }
    if (threads > max_threads) return set_error(B200_ERR_INVALID, "tile volume %d exceeds %d threads", threads, max_threads);
    return 0;
  }

  // grid of a box launch; returns false if the box is empty
  inline bool box_grid(TileMap &tm, int n_parity, int &gx, int &gy, int &gz, int &rc)
  {
    rc = 0;
    for (int d = 0; d < 4; d++)
      if (tm.cnt[d] <= 0) return false;
    tm.cnt0_magic = tm.cnt[0] >= 2 ? (unsigned)(0x100000000ull / (unsigned)tm.cnt[0]) + 1u : 0u;
    // umulhi(b, magic) == b / cnt0 needs b * cnt0 < 2^32
    if ((long long)tm.cnt[0] * tm.cnt[0] * tm.cnt[1] >= (1ll << 32) || tm.cnt[2] > 65535 || tm.cnt[3] * n_parity > 65535) {
      rc = set_error(B200_ERR_INVALID, "lattice too large for the tile grid");
      return false;
    }
    gx = tm.cnt[0] * tm.cnt[1];
    gy = tm.cnt[2];
    gz = tm.cnt[3] * n_parity;
    return true;
  }

  // Split the tiles of a partitioned lattice into the box that touches no partitioned face (tm.org / tm.cnt) and a
  // disjoint set of boundary slabs: going from the highest partitioned dimension down, the slab(s) of dimension D fix
  // the tile index of D to its first / last value, take the interior range in the partitioned dimensions above D and
  // the full range everywhere else.  Returns the number of boundary CTAs.
  inline int split_boundary(TileMap &tm, SlabTable &st, const int *comm_dim)
  {
    st.n = 0;
    st.cta_start[0] = 0;
    for (int d = 0; d < 4; d++) {
      tm.org[d] = comm_dim[d] ? 1 : 0;
      tm.cnt[d] = tm.nt[d] - (comm_dim[d] ? 2 : 0); // <= 0: no interior tile at all in that dimension
    }
    for (int D = 3; D >= 0; D--) {
      if (!comm_dim[D]) continue;
      const int nb = tm.nt[D] >= 2 ? 2 : 1;
      for (int k = 0; k < nb; k++) {
        int org[4], cnt[4];
        long ctas = 1;
        for (int e = 0; e < 4; e++) {
          if (e == D) {
            org[e] = k == 0 ? 0 : tm.nt[D] - 1;
            cnt[e] = 1;
          } else if (e > D && comm_dim[e]) {
            org[e] = 1;
            cnt[e] = tm.nt[e] - 2;
          } else {
            org[e] = 0;
            cnt[e] = tm.nt[e];
          }
          ctas *= cnt[e] > 0 ? cnt[e] : 0;
        }
        if (ctas <= 0) continue;
        for (int e = 0; e < 4; e++) {
          st.org[st.n][e] = org[e];
          st.cnt[st.n][e] = cnt[e];
        }
        st.cta_start[st.n + 1] = st.cta_start[st.n] + (int)ctas;
        st.n++;
      }
    }
    return st.cta_start[st.n];
  }

  // tile box of a multi-RHS launch: every tile, or -- partitioned lattice -- the tiles that touch no partitioned face
  // (what dslash_interior_kernel covers for B200_KERNEL_INTERIOR_TILES, same tiling, so the per-source boundary launches
  // complete the lattice exactly).  Returns false with rc == 0 if there is nothing to launch.
  inline bool mrhs_box(TileMap &tm, const MrhsRequest &rq, const int *comm_dim, int n_parity, int &gx, int &gy, int &gz, int &rc)
  {
    if (rq.interior_box) {
      SlabTable st;
      split_boundary(tm, st, comm_dim);
    }
    if (box_grid(tm, n_parity, gx, gy, gz, rc)) return true;
    if (!rc && !rq.interior_box) rc = set_error(B200_ERR_INVALID, "empty lattice");
    return false;
  }

  template <class P> int launch_precision(const LaunchRequest &rq);
  constexpr int kTmaSkip = -4242; // "this request is not served by the TMA kernel": the caller uses the gather kernel
  template <class P> int launch_tma_precision(const LaunchRequest &rq); // tma_kernel.cuh; kTmaSkip if not served
  template <class P> int launch_mrhs_precision(const MrhsRequest &rq);
  template <class P> int launch_clover_precision(const CloverRequest &rq);
  template <class P> int launch_twist_precision(const TwistRequest &rq);
  template <class P> int launch_pack_precision(const PackRequest &rq);
  template <class P> int launch_pack_multi_precision(const PackRequest &rq, const PackBatchRequest &batch);
  template <class P> int launch_copy_precision(const CopyRequest &rq);
  template <class P> int launch_gauge_copy_precision(const GaugeCopyRequest &rq);
  template <class P> int launch_clover_copy_precision(const CloverCopyRequest &rq);

} // namespace b200
