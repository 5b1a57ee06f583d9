// TEST-ONLY "host twin": the library's entry points with a CPU executor.  Its twin_* functions forward to the same
// templates as libquda_b200's b200_* functions (quda_b200/csrc/plan.h: argument validation, environment knobs,
// orchestration, template dispatch and launch plans); the executor below walks every planned launch grid block by block
// and thread by thread and runs the product's site code (dslash_site.h, core.h, clover.h -- the exact functions the CUDA
// kernels call) in plain CPU loops.  It exists so that the launch logic, layouts, gauge reconstruction, fixed-point
// handling, clover compression and the halo index maps can be checked against the CPU oracle in the CPU-only test tier.
// It is NOT part of the product: nothing under quda_b200/ loads it, and libquda_b200.so has no CPU path.
#include <cstdarg>
#include <cstdio>
#include <numeric>
#include <type_traits>
#include <vector>

#include "../../quda_b200/csrc/plan.h"
#include "tma_emu.h"

namespace b200
{
  static char g_err[512] = "";
  int set_error(int code, const char *fmt, ...)
  {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
    return code;
  }
  int check_cuda(cudaError_t, const char *) { return 0; }
  void count_launch() { }

  constexpr int kH100Sms = 132; // CTAs of the TMA kernel's persistent grid on an H100 (one per SM)

  // kernels.cuh::wait_for_halo: every role that reads ghost zones first acquires the arrival counters.  The twin runs
  // pack and Dslash one after the other, so a counter below its target is a deadlock (or a 10 s timeout) on the GPU.
  template <class Arg> int check_halo_arrived(const Arg &arg)
  {
    const unsigned uses = (arg.seq + (arg.seq & 1u)) >> 1;
    for (int d = 0; d < 4; d++)
      for (int dir = 0; dir < 2; dir++)
        if (const unsigned *f = arg.wait_flag[d][dir]) {
          const unsigned target = uses * (unsigned)arg.geom.face_cb[d];
          if ((int)(*f - target) < 0)
            return set_error(B200_ERR_INVALID, "halo wait would never finish: counter[%d][%d] = %u < %u (exchange %u)", d, dir, *f, target, arg.seq);
        }
    return 0;
  }

  // A pack grid CTA by CTA in a scrambled order (CTAs retire in any order on the GPU).  cta(c, face_id, blk, nblk, views)
  // describes CTA c (false: it has no work): its `block` threads run pack_site, then the ticket protocol of
  // kernels.cuh::pack_block follows -- the CTA that draws ticket nblk - 1 of its face publishes the arrival count.  Checks
  // on the way that the count is published exactly once per face and only after every site of all `n_src` sources landed.
  template <class P, class Cta> int walk_pack(const PackArgs<P> &arg, long n_cta, int block, int n_src, Cta &&cta)
  {
    const Geom &g = arg.geom;
    int tickets[8] = {0}, published[8] = {0};
    long written[8] = {0};
    // an odd multiplier coprime to n_cta visits every CTA exactly once in a scrambled order
    long mul = 7919;
    while (std::gcd(mul, n_cta) != 1) mul += 2;
    for (long k = 0; k < n_cta; k++) {
      int f, blk, nblk;
      PackSourceViews<P> vw;
      if (!cta((k * mul + 12345) % n_cta, f, blk, nblk, vw)) continue;
      const int d = f >> 1, face = f & 1;
      for (int tid = 0; tid < block; tid++) {
        const int idx = blk * block + tid;
        if (idx >= g.face_cb[d]) continue;
        pack_site(arg, vw, d, face, idx);
        written[f]++;
      }
      if (unsigned *sig = arg.signal[d][face]) {
        const int prev = tickets[f]++;
        if (prev == nblk - 1) {
          if (written[f] != (long)n_src * g.face_cb[d]) return set_error(B200_ERR_INVALID, "face %d signalled before all sources landed", f);
          if (published[f]++) return set_error(B200_ERR_INVALID, "face %d signalled twice", f);
          tickets[f] = 0;
          *sig = ((arg.seq + (arg.seq & 1u)) >> 1) * (unsigned)g.face_cb[d];
        }
      }
    }
    for (int f = 0; f < 8; f++)
      if (arg.signal[f >> 1][f & 1] && published[f] != 1) return set_error(B200_ERR_INVALID, "face %d never signalled", f);
    return 0;
  }

  // one planned Dslash (plan.h::plan_dslash), launch by launch as kernels.cuh::launch_config issues it.  Counts the site
  // updates on the way: no launch plan may update a site twice, and a plan for the whole operator updates every one.
  template <class P, int recon, bool dagger, bool xpay, OpType op>
  int run_config(OpCfg<dagger, xpay, op>, const LaunchRequest &rq, const DslashArgs<P, recon> &arg)
  {
    LaunchPlan pl;
    if (int rc = plan_dslash(pl, rq, arg)) return rc;
    const Geom &g = arg.geom;
    std::vector<int> hits(2 * (size_t)g.volume_cb, 0);
    auto twice = [&](int par, int x_cb) -> long {
      int prev;
#pragma omp atomic capture
      prev = hits[(size_t)par * g.volume_cb + x_cb]++;
      return prev != 0;
    };
    // dslash_interior_kernel<..., part> over the box of step l
    auto interior = [&](const LaunchStep &l, auto part) {
      long rep = 0;
#pragma omp parallel for collapse(2) reduction(+ : rep)
      for (int bz = 0; bz < l.grid[2]; bz++)
        for (int by = 0; by < l.grid[1]; by++)
          for (int bx = 0; bx < l.grid[0]; bx++)
            for (int tid = 0; tid < l.threads; tid++) {
              int x[4], x_cb, par;
              if (!tile_site(x, x_cb, par, g, l.tm, arg.n_parity, arg.parity, bx, by, bz, tid)) continue;
              dslash_site_interior<P, recon, dagger, xpay, op, decltype(part)::value>(arg, x, x_cb, par);
              rep += twice(par, x_cb);
            }
      return rep;
    };
    long repeats = 0;
    for (int i = 0; i < pl.n; i++) {
      const LaunchStep &l = pl.step[i];
      if (l.kind == LAUNCH_INTERIOR && !l.masked) {
        repeats += interior(l, std::false_type {});
      } else if constexpr (!has_partitioned_kernels(op)) {
        return refuse_partitioned_tm_pc_pre();
      } else if (l.kind == LAUNCH_INTERIOR) {
        repeats += interior(l, std::true_type {});
      } else if (l.kind == LAUNCH_FUSED) {
        // dslash_fused_kernel: the pack CTAs first (all faces land before any boundary CTA waits), then blocks n_pack + b
        const FusedShape &fs = l.fs;
        if (fs.n_pack) {
          PackArgs<P> pk;
          fill_pack_args(pk, *rq.fused_pack);
          const int rc = walk_pack(pk, fs.n_pack, l.threads, 1, [&](long c, int &f, int &blk, int &nblk, PackSourceViews<P> &vw) {
            const int b = (int)c;
            f = fused_pack_face(fs, b);
            blk = b - fs.pack_start[f];
            nblk = fs.pack_start[f + 1] - fs.pack_start[f];
            vw = PackSourceViews<P> {pk.in, pk.dst[f >> 1][f & 1]};
            return true;
          });
          if (rc) return rc;
        }
        if (fs.n_boundary)
          if (int rc = check_halo_arrived(arg)) return rc;
#pragma omp parallel for reduction(+ : repeats)
        for (int b = 0; b < l.grid[0] - fs.n_pack; b++) {
          const int ib = fused_interior_tile(fs, b);
          int bx = 0, by = 0, bz = 0;
          if (ib >= 0) fused_tile_block(fs, ib, bx, by, bz);
          for (int tid = 0; tid < l.threads; tid++) {
            int x[4], x_cb, par = arg.parity;
            if (ib >= 0) {
              if (!tile_site(x, x_cb, par, g, l.tm, arg.n_parity, arg.parity, bx, by, bz, tid) || !site_is_interior(arg, x)) continue;
              dslash_site_interior<P, recon, dagger, xpay, op, false>(arg, x, x_cb, par);
            } else {
              const int t = (b - fs.n_interior_first) * l.threads + tid;
              if (t >= arg.threads_ext[4] || !exterior_thread_site(x, x_cb, arg, t, par)) continue;
              dslash_site_full<P, recon, dagger, xpay, op>(arg, x, x_cb, par);
            }
            repeats += twice(par, x_cb);
          }
        }
      } else {
        if (int rc = check_halo_arrived(arg)) return rc;
        for (int by = 0; by < l.grid[1]; by++) {
          const int par = arg.n_parity == 2 ? by : arg.parity;
#pragma omp parallel for reduction(+ : repeats)
          for (int bx = 0; bx < l.grid[0]; bx++)
            for (int tid = 0; tid < l.threads; tid++) {
              int x[4], x_cb;
              if (l.kind == LAUNCH_BOUNDARY) {
                if (!slab_site(x, x_cb, g, l.tm, l.st, par, bx, tid)) continue;
                dslash_site_full<P, recon, dagger, xpay, op>(arg, x, x_cb, par);
              } else {
                const int t = bx * l.threads + tid;
                if (t >= arg.threads_ext[4] || !exterior_thread_site(x, x_cb, arg, t, par)) continue;
                dslash_site_exterior<P, recon, dagger, xpay, op>(arg, x, x_cb, par);
              }
              repeats += twice(par, x_cb);
            }
        }
      }
    }
    if (repeats) return set_error(B200_ERR_INVALID, "the launch plan updates %ld sites more than once", repeats);
    const long updated = std::accumulate(hits.begin(), hits.end(), 0L), all = (long)g.volume_cb * arg.n_parity;
    if (pl.whole && updated != all) return set_error(B200_ERR_INVALID, "the launch plan updates %ld of %ld sites", updated, all);
    return 0;
  }

  // one multi-RHS launch as mrhs.cuh issues it: the CTA flavour (NS == 0: blockIdx.x = tile * n_batch + batch, threadIdx =
  // (site in tile, source in CTA)) or NS sources per thread from source s0 on
  template <int NS, class P, int recon, bool dagger, bool xpay, OpType op>
  int run_mrhs(OpCfg<dagger, xpay, op>, const MrhsRequest &rq, const DslashArgs<P, recon> &arg, int s0)
  {
    MrhsGrid m;
    if (int rc = plan_mrhs(m, rq, arg, NS == 0)) return rc;
    if (!m.gx) return 0;
    MrhsViews<P> views;
    MrhsFields<P, NS ? NS : 1> fields;
    if constexpr (NS == 0)
      fill_mrhs_views(views, rq);
    else
      fill_mrhs_fields(fields, rq, s0);
    const Geom &g = arg.geom;
    long visited = 0;
#pragma omp parallel for collapse(2) reduction(+ : visited)
    for (int bz = 0; bz < m.gz; bz++)
      for (int by = 0; by < m.gy; by++)
        for (int bx = 0; bx < m.gx * m.n_batch; bx++)
          for (int ty = 0; ty < m.nsb; ty++)
            for (int tid = 0; tid < m.threads; tid++) {
              const unsigned tile = (unsigned)bx / (unsigned)m.n_batch;
              const int s = (bx - (int)tile * m.n_batch) * m.nsb + ty;
              if (s >= rq.n_src) continue;
              int x[4], x_cb, par;
              if (!tile_site(x, x_cb, par, g, m.tm, arg.n_parity, arg.parity, tile, by, bz, tid)) continue;
              if constexpr (NS == 0)
                dslash_site_src<P, recon, dagger, xpay, op, Cache::REUSE>(arg, views.in[s][1 - par], views.out[s][par], views.x[s][par], x, x_cb, par);
              else
                dslash_site_mrhs<P, recon, dagger, xpay, op, NS>(arg, fields, x, x_cb, par);
              visited++;
            }
    const long want = (long)g.volume_cb * arg.n_parity * (NS == 0 ? rq.n_src : 1);
    if (!rq.interior_box && visited != want) return set_error(B200_ERR_INVALID, "multi-RHS grid visited %ld of %ld (site, source) pairs", visited, want);
    return 0;
  }

  // the executor of plan.h's entry points: CPU walkers of the launch grids the CUDA launchers issue
  struct Twin {
    static int require_device() { return 0; }

    template <class P> static int dslash(const LaunchRequest &rq)
    {
      return dispatch_dslash<P>(rq, [&](auto c, const auto &arg) { return run_config(c, rq, arg); });
    }

    template <class P> static int tma(const LaunchRequest &rq)
    {
      return dispatch_tma<P>(rq, [&](auto c, const auto &arg) { return tma_emu_launch(c, rq, arg, kH100Sms); });
    }

    template <class P> static int mrhs(const MrhsRequest &rq)
    {
      return dispatch_mrhs<P>(rq, [&](auto c, const auto &arg, auto ns, int s0) -> int {
        constexpr int NS = decltype(ns)::value;
        if constexpr (NS == 1)
          return dslash<P>(mrhs_source(rq, s0));
        else
          return run_mrhs<NS>(c, rq, arg, s0);
      });
    }

    // clover_apply_kernel / twist_gamma5_kernel: one thread per site
    template <class P> static int clover(const CloverRequest &rq)
    {
      SpinorView<P> out, in;
      CloverView<P> A;
      fill_spinor(out, rq.out, rq.out_norm, rq.volume_cb);
      fill_spinor(in, rq.in, rq.in_norm, rq.volume_cb);
      fill_clover(A, rq.A, rq.volume_cb);
      for (int x_cb = 0; x_cb < rq.volume_cb; x_cb++) {
        typename P::real v[24];
        in.load(v, x_cb);
        if (rq.inverse)
          clover_apply_site<P, true>(v, A, x_cb, rq.parity);
        else
          clover_apply_site<P, false>(v, A, x_cb, rq.parity);
        out.save(v, x_cb);
      }
      return 0;
    }

    template <class P> static int twist(const TwistRequest &rq)
    {
      SpinorView<P> out, in;
      fill_spinor(out, rq.out, rq.out_norm, rq.volume_cb);
      fill_spinor(in, rq.in, rq.in_norm, rq.volume_cb);
      for (int x_cb = 0; x_cb < rq.volume_cb; x_cb++) {
        typename P::real v[24];
        in.load(v, x_cb);
        twist_apply(v, (typename P::real)rq.a, (typename P::real)rq.b);
        out.save(v, x_cb);
      }
      return 0;
    }

    // pack_multi_kernel: grid (blocks over the largest face, 8 face ids, n_src sources) of 128 threads
    template <class P> static int pack_multi(const PackRequest &rq, const PackBatchRequest &b)
    {
      int gx;
      if (int rc = pack_blocks(gx, rq)) return rc;
      if (!gx) return 0;
      PackArgs<P> arg;
      fill_pack_args(arg, rq);
      PackBatch<P> batch;
      fill_pack_batch(batch, b, arg.geom.volume_cb);
      return walk_pack(arg, (long)gx * 8 * b.n_src, 128, b.n_src, [&](long c, int &f, int &blk, int &nblk, PackSourceViews<P> &vw) {
        blk = (int)(c % gx);
        f = (int)((c / gx) % 8);
        const int s = (int)(c / ((long)gx * 8)), d = f >> 1;
        const int n = (arg.geom.face_cb[d] + 127) / 128;
        if (!arg.comm_dim[d] || blk >= n) return false;
        nblk = n * batch.n_src;
        vw = PackSourceViews<P> {arg.in, ghost_of_source(arg.dst[d][f & 1], (size_t)s * batch.dst_stride[d])};
        vw.in_.v = batch.in[s];
        vw.in_.norm = batch.in_norm[s];
        return true;
      });
    }

    // pack_kernel: the same grid with one source, its own field
    template <class P> static int pack(const PackRequest &rq)
    {
      PackBatchRequest one {};
      one.n_src = 1;
      one.in[0] = rq.in;
      one.in_norm[0] = rq.in_norm;
      return pack_multi<P>(rq, one);
    }
  };
} // namespace b200

using namespace b200;

extern "C" {
const char *twin_last_error(void) { return g_err; }

int twin_dslash_apply(const b200_dslash_args *a) { return apply_dslash<Twin>(a); }

int twin_dslash_apply_fused(const b200_dslash_args *a, const b200_pack_args *p) { return apply_dslash_fused<Twin>(a, p); }

int twin_dslash_apply_multi(const b200_dslash_args *a, int n_src, const b200_spinor *out, const b200_spinor *in, const b200_spinor *x)
{
  return apply_dslash_multi<Twin>(a, n_src, out, in, x);
}

int twin_clover_apply(const b200_spinor *out, const b200_spinor *in, const b200_clover *A, int precision, int inverse, int parity, void *stream)
{
  return clover_apply<Twin>(out, in, A, precision, inverse, parity, stream);
}

int twin_twist_gamma5(const b200_spinor *out, const b200_spinor *in, int precision, double kappa, double mu, int dagger, int inverse, void *stream)
{
  return twist_gamma5<Twin>(out, in, precision, kappa, mu, dagger, inverse, stream);
}

int twin_pack_ghost_multi(const b200_pack_args *a, int n_src, const b200_spinor *in, const size_t dst_stride[4])
{
  return pack_ghost_multi<Twin>(a, n_src, in, dst_stride);
}

int twin_pack_ghost(const b200_pack_args *a) { return pack_ghost<Twin>(a); }
}
