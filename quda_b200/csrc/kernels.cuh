// __global__ wrappers around the site functions + the per-precision launchers that issue plan.h's launch plans.
// One translation unit per storage precision includes this header (inst_f64.cu, inst_f32.cu, inst_h16.cu)
// so the three compile in parallel.
#pragma once

#include <cstdlib>
#include <cuda_runtime.h>

#include "dslash_site.h"
#include "plan.h"

namespace b200
{

  // Occupancy targets per storage precision: CTAs hold at most B2_MAXTILE threads (the default tiles are
  // 64..128 threads: full x rows x a few y/z rows) and ptxas may use 65536 / (B2_MAXTILE * minBlocks) registers per
  // thread.  The stencil is latency bound (ncu: long-scoreboard stalls dominate), so registers spent on keeping the
  // loads of several hops in flight pay better than extra resident warps: fp64 255 regs, fp32 128, half 128.
#ifndef B2_MINBLOCKS_F64
#define B2_MINBLOCKS_F64 2
#endif
#ifndef B2_MINBLOCKS_F32
#define B2_MINBLOCKS_F32 4
#endif
#ifndef B2_MINBLOCKS_H16
#define B2_MINBLOCKS_H16 4
#endif
  template <class P> struct MinBlocks { static constexpr int value = B2_MINBLOCKS_F32; };
  template <> struct MinBlocks<PrecF64> { static constexpr int value = B2_MINBLOCKS_F64; };
  template <> struct MinBlocks<PrecH16> { static constexpr int value = B2_MINBLOCKS_H16; };

  // Optional L2 look-ahead: the first thread of every 128-byte line segment asks L2 for the links (and the input
  // spinor) of the tile that a CTA B2_L2_PREFETCH launch slots further on will work on, so that by the time those
  // CTAs run their link loads are L2 hits instead of full DRAM round trips.  The links are 2/3 of the traffic and a
  // pure stream, i.e. perfectly predictable.
#ifndef B2_L2_PREFETCH
#define B2_L2_PREFETCH 0
#endif
  __device__ __forceinline__ void prefetch_l2(const void *p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

  template <class P, int recon>
  __device__ __forceinline__ void prefetch_future_tile(const DslashArgs<P, recon> &arg, const TileMap &tm)
  {
    using GV = GaugeView<P, recon>;
    constexpr int lanes_per_line = 128 / sizeof(typename GV::V);
    if ((threadIdx.x & ((1 << tm.sh[0]) - 1)) % lanes_per_line != 0) return;
    const unsigned gx = gridDim.x, gy = gridDim.y, gz = gridDim.z;
    unsigned lin = blockIdx.x + gx * (blockIdx.y + gy * blockIdx.z) + B2_L2_PREFETCH;
    if (lin >= gx * gy * gz) return;
    const unsigned bz = lin / (gx * gy);
    lin -= bz * gx * gy;
    const unsigned by = lin / gx;
    const unsigned bx = lin - by * gx;
    int x[4], x_cb, parity;
    if (!tile_site(x, x_cb, parity, arg.geom, tm, arg.n_parity, arg.parity, bx, by, bz, threadIdx.x)) return;
    const Geom &g = arg.geom;
    const typename GV::V *gf = reinterpret_cast<const typename GV::V *>(arg.U.g[parity]);
    const typename GV::V *gb = reinterpret_cast<const typename GV::V *>(arg.U.g[1 - parity]);
#pragma unroll
    for (int d = 0; d < 4; d++) {
      int y[4] = {x[0], x[1], x[2], x[3]};
      y[d] = (x[d] - 1 < 0) ? g.X[d] - 1 : x[d] - 1;
      const int n_cb = cb_from_coords(y, g);
#pragma unroll
      for (int i = 0; i < GV::M; i++) {
        prefetch_l2(gf + (size_t)(d * GV::M + i) * arg.U.stride + x_cb);
        prefetch_l2(gb + (size_t)(d * GV::M + i) * arg.U.stride + n_cb);
      }
    }
  }

  // `part` == false: no dimension is partitioned -> the stencil is completely branch free
  template <class P, int recon, bool dagger, bool xpay, OpType op, bool part>
  __global__ void __launch_bounds__(kMaxTile, MinBlocks<P>::value)
    dslash_interior_kernel(const __grid_constant__ DslashArgs<P, recon> arg, const __grid_constant__ TileMap tm)
  {
    if constexpr (B2_L2_PREFETCH > 0) prefetch_future_tile(arg, tm);
    int x[4], x_cb, parity;
    if (!tile_site(x, x_cb, parity, arg.geom, tm, arg.n_parity, arg.parity, blockIdx.x, blockIdx.y, blockIdx.z, threadIdx.x))
      return;
    dslash_site_interior<P, recon, dagger, xpay, op, part>(arg, x, x_cb, parity);
  }

  // ---- system-scope flag helpers for the NVLink remote-write halo path (used by the kernels below)
  __device__ __forceinline__ unsigned ld_acquire_sys(const unsigned *p)
  {
    unsigned v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
  }
  __device__ __forceinline__ void st_release_sys(unsigned *p, unsigned v)
  {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
  }
  __device__ __forceinline__ void red_release_sys_add(unsigned *p, unsigned v)
  {
    asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
  }

  // Block until every partitioned face of exchange `seq` has arrived.  A flag word counts the face sites its buffer has
  // received since the exchange was created; buffer b = seq & 1 is used by every second exchange, so exchange `seq` is
  // complete once the count reaches ((seq + b) / 2) * face_cb[d] (compared wrap-safe).  One thread polls, the CTA follows.
  // Gives up after ~10 s of SM clock so that a lost peer can never hang the GPU; the host layer checks (and clears)
  // timeout_flag at its synchronisation points and turns it into an error (b200_comm_check, b200_invert_cg).
  template <class Arg> __device__ __forceinline__ void wait_for_halo(const Arg &arg)
  {
    if (threadIdx.x == 0) {
      const long long t0 = clock64();
      const unsigned uses = (arg.seq + (arg.seq & 1u)) >> 1;
#pragma unroll
      for (int d = 0; d < 4; d++) {
#pragma unroll
        for (int dir = 0; dir < 2; dir++) {
          const unsigned *f = arg.wait_flag[d][dir];
          if (!f) continue;
          const unsigned target = uses * (unsigned)arg.geom.face_cb[d];
          while ((int)(ld_acquire_sys(f) - target) < 0) {
            if (clock64() - t0 > 20000000000LL) {
              if (arg.timeout_flag) *arg.timeout_flag = 1;
              break;
            }
            __nanosleep(100);
          }
        }
      }
    }
    __syncthreads();
  }

  // Boundary tiles: wait for the neighbours' faces, then update the sites completely (local + ghost hops, clover, xpay)
  template <class P, int recon, bool dagger, bool xpay, OpType op>
  __global__ void __launch_bounds__(kMaxTile, MinBlocks<P>::value)
    dslash_boundary_kernel(const __grid_constant__ DslashArgs<P, recon> arg, const __grid_constant__ TileMap tm,
                           const __grid_constant__ SlabTable st)
  {
    wait_for_halo(arg);
    const int parity = arg.n_parity == 2 ? blockIdx.y : arg.parity;
    int x[4], x_cb;
    if (!slab_site(x, x_cb, arg.geom, tm, st, parity, blockIdx.x, threadIdx.x)) return;
    dslash_site_full<P, recon, dagger, xpay, op>(arg, x, x_cb, parity);
  }

  template <class P, int recon, bool dagger, bool xpay, OpType op>
  __global__ void __launch_bounds__(256) dslash_exterior_kernel(const __grid_constant__ DslashArgs<P, recon> arg)
  {
    wait_for_halo(arg);
    const int parity = arg.n_parity == 2 ? blockIdx.y : arg.parity;
    const int tid = blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= arg.threads_ext[4]) return;
    int x[4], x_cb;
    if (!exterior_thread_site(x, x_cb, arg, tid, parity)) return;
    dslash_site_exterior<P, recon, dagger, xpay, op>(arg, x, x_cb, parity);
  }

  template <class P, bool inverse>
  __global__ void __launch_bounds__(256) clover_apply_kernel(SpinorView<P> out, SpinorView<P> in, CloverView<P> A,
                                                             int volume_cb, int parity)
  {
    const int x_cb = blockIdx.x * blockDim.x + threadIdx.x;
    if (x_cb >= volume_cb) return;
    typename P::real v[24];
    in.template load<Cache::COHERENT>(v, x_cb); // `out` may be `in` (in-place apply): not the .nc path
    clover_apply_site<P, inverse>(v, A, x_cb, parity);
    out.save(v, x_cb);
  }

  // site-local twisted-mass rotation out = a (1 + i b gamma5) in (ApplyTwistGamma, dslash_gamma_helper.cuh)
  template <class P>
  __global__ void __launch_bounds__(256) twist_gamma5_kernel(SpinorView<P> out, SpinorView<P> in, int volume_cb,
                                                             typename P::real a, typename P::real b)
  {
    const int x_cb = blockIdx.x * blockDim.x + threadIdx.x;
    if (x_cb >= volume_cb) return;
    typename P::real v[24];
    in.template load<Cache::COHERENT>(v, x_cb); // `out` may be `in`
    twist_apply(v, a, b);
    out.save(v, x_cb);
  }

  // Halo packing: one thread per (dim, face, face site) runs plan.h::pack_site, which stores the projected half spinor
  // to the destination face buffer (local, or a peer GPU's ghost buffer mapped over NVLink).
#ifndef B2_PACK_REMOTE_ADD
#define B2_PACK_REMOTE_ADD 0
#endif
  // one CTA of the pack: sites [blk * blockDim.x, ...) of face `face_id` = 2*d + face; `nblk` CTAs (of all sources of a
  // batch together) work on this face before its arrival counter moves
  template <class P, class Views>
  __device__ __forceinline__ void pack_block(const PackArgs<P> &arg, const Views &vw, int face_id, int blk, int nblk)
  {
    const Geom &g = arg.geom;
    const int d = face_id >> 1, face = face_id & 1;
    const int idx = blk * blockDim.x + threadIdx.x;
    if (idx < g.face_cb[d]) pack_site(arg, vw, d, face, idx);
    unsigned *sig = arg.signal[d][face];
    if (sig) {
      // Arrival protocol: the flag word in the RECEIVER's memory holds the number of face sites that have landed in this
      // buffer since the exchange was created; exchange `seq` is complete at ((seq + (seq & 1)) / 2) * face_cb.
      // Per CTA: barrier (orders every thread's possibly remote stores before thread 0), ONE system fence by thread 0, then
      // a LOCAL ticket; the CTA that draws the last ticket publishes the new total with a single remote store.  (Round 1
      // fenced in every thread -- MEMBAR.SYS was the hottest instruction of the fused launch, profiles/r02_fused_self_*; one
      // remote release-add per CTA avoids the tickets but serialises 512 NVLink atomics on one address: 111 us per step at
      // 2 GPUs, profiles/r02_scale2_remote_add.json.)
      __syncthreads();
      if (threadIdx.x == 0) {
#if B2_PACK_REMOTE_ADD
        const int left = g.face_cb[d] - blk * (int)blockDim.x;
        red_release_sys_add(sig, (unsigned)(left < (int)blockDim.x ? left : (int)blockDim.x));
#else
        __threadfence_system();
        const int prev = atomicAdd(arg.counter + face_id, 1);
        if (prev == nblk - 1) {
          arg.counter[face_id] = 0;
          __threadfence_system();
          const unsigned uses = (arg.seq + (arg.seq & 1u)) >> 1;
          st_release_sys(sig, uses * (unsigned)g.face_cb[d]);
        }
#endif
      }
    }
  }

  template <class P> __device__ __forceinline__ void pack_block(const PackArgs<P> &arg, int face_id, int blk, int nblk)
  {
    pack_block(arg, PackOwnViews<P> {arg}, face_id, blk, nblk);
  }

  // grid: x = blocks over the largest face, y = face id (2*d + face)
  template <class P> __global__ void __launch_bounds__(128) pack_kernel(const __grid_constant__ PackArgs<P> arg)
  {
    const int d = blockIdx.y >> 1;
    if (!arg.comm_dim[d]) return;
    const int nblk = (arg.geom.face_cb[d] + blockDim.x - 1) / blockDim.x;
    if ((int)blockIdx.x >= nblk) return;
    pack_block(arg, blockIdx.y, blockIdx.x, nblk);
  }

  // Batched (multi-RHS) pack: the faces of ALL sources of a cvector_ref batch leave in one launch and raise ONE arrival
  // signal per face (reference: lib/dslash_pack2.cu:55-403 packs every source of the batch in one kernel, the source index
  // riding in the thread grid).  grid.z = source; source s reads batch.in[s] and writes s * dst_stride[d] bytes behind the
  // first source's slab.  The tickets count the CTAs of all sources, so the counter in the receiver's memory moves -- to
  // the same value as for a single exchange `seq` -- only when the last source's last site has landed; each source's
  // boundary kernel then waits on that one counter and reads its own slab.
  template <class P>
  __global__ void __launch_bounds__(128) pack_multi_kernel(const __grid_constant__ PackArgs<P> arg, const __grid_constant__ PackBatch<P> batch)
  {
    static_assert(!B2_PACK_REMOTE_ADD, "the batched pack relies on the ticket protocol");
    const int d = blockIdx.y >> 1, face = blockIdx.y & 1;
    if (!arg.comm_dim[d]) return;
    const int nblk = (arg.geom.face_cb[d] + blockDim.x - 1) / blockDim.x;
    if ((int)blockIdx.x >= nblk) return;
    const int s = blockIdx.z;
    PackSourceViews<P> vw {arg.in, ghost_of_source(arg.dst[d][face], (size_t)s * batch.dst_stride[d])};
    vw.in_.v = batch.in[s];
    vw.in_.norm = batch.in_norm[s];
    pack_block(arg, vw, blockIdx.y, blockIdx.x, nblk * batch.n_src);
  }

  // ------------------------------------------------------------------ ONE launch per partitioned Dslash
  // The reference overlaps halo and interior with a policy of several kernels on several streams plus host-side event
  // plumbing (lib/dslash_policy.hpp:1471-1650; pack CTAs folded into the interior launch: include/dslash_helper.cuh:664-713).
  // Here the whole partitioned Dslash is one grid whose block index selects the role:
  //   [0, n_pack)                 pack CTAs: spin-project the face sites and write them straight into the neighbours'
  //                               ghost slabs over NVLink; the last CTA of a face raises the arrival flag there
  //   [n_pack, n_pack + n_int)    interior CTAs: the branch-free stencil on every site that touches no partitioned face
  //                               (threads of face sites retire at once) -- independent of the halo
  //   boundary CTAs               one thread per face site (corner sites owned by the highest partitioned dimension),
  //                               acquire the neighbours' arrival counters, then update the site completely; they sit
  //                               behind the first ~70 % of the interior CTAs (B200_FUSED_BOUNDARY_AT) and in front of the
  //                               rest, so their wait + latency is covered by interior work instead of forming a tail
  // Blocks are dispatched in index order, so the faces leave first and the interior streams while they fly.  No second
  // stream, no events, no exterior read-modify-write pass.  The host twin decodes block indices with plan.h's
  // fused_pack_face / fused_interior_tile / fused_tile_block; calling them here changes this kernel's machine code, so
  // it keeps its own copy of the decode -- change both together.
  template <class P, int recon, bool dagger, bool xpay, OpType op>
  __global__ void __launch_bounds__(kMaxTile, MinBlocks<P>::value)
    dslash_fused_kernel(const __grid_constant__ DslashArgs<P, recon> arg, const __grid_constant__ TileMap tm,
                        const __grid_constant__ PackArgs<P> pk, const __grid_constant__ FusedShape fs)
  {
    int b = blockIdx.x;
    if (b < fs.n_pack) {
      int f = 0;
#pragma unroll
      for (int k = 1; k < 8; k++)
        if (b >= fs.pack_start[k]) f = k;
      pack_block(pk, f, b - fs.pack_start[f], fs.pack_start[f + 1] - fs.pack_start[f]);
      return;
    }
    b -= fs.n_pack;
    // block order after the pack CTAs: [interior part 1 | boundary | interior part 2] -- the boundary CTAs start when most of
    // the interior is already in flight (by then the neighbours' faces have landed) and their latency is covered by the rest
    // of the interior instead of forming the tail of the launch
    int ib = -1;
    if (b < fs.n_interior_first)
      ib = b;
    else if (b >= fs.n_interior_first + fs.n_boundary)
      ib = b - fs.n_boundary;
    if (ib >= 0) {
      const int per_z = fs.gx * fs.gy;
      const int bz = ib / per_z;
      const int r = ib - bz * per_z;
      const int by = r / fs.gx;
      const int bx = r - by * fs.gx;
      int x[4], x_cb, parity;
      if (!tile_site(x, x_cb, parity, arg.geom, tm, arg.n_parity, arg.parity, bx, by, bz, threadIdx.x)) return;
      if (!site_is_interior(arg, x)) return;
      dslash_site_interior<P, recon, dagger, xpay, op, false>(arg, x, x_cb, parity);
      return;
    }
    b -= fs.n_interior_first;
    wait_for_halo(arg);
    const int tid = b * blockDim.x + threadIdx.x;
    if (tid >= arg.threads_ext[4]) return;
    int x[4], x_cb;
    if (!exterior_thread_site(x, x_cb, arg, tid, arg.parity)) return;
    dslash_site_full<P, recon, dagger, xpay, op>(arg, x, x_cb, arg.parity);
  }

  // Host interface order <-> native order, with the DeGrand-Rossi <-> UKQCD rotation
  // out[s] = K1[s] in[s1[s]] + K2[s] in[s2[s]], s1 = {1,2,3,0}, s2 = {3,0,1,2} (copy_color_spinor.cuh:51-89)
  template <class P, typename H, bool to_native>
  __global__ void __launch_bounds__(128) copy_spinor_kernel(SpinorView<P> nat, H *host, int volume_cb)
  {
    using real = typename P::real;
    const int x_cb = blockIdx.x * blockDim.x + threadIdx.x;
    if (x_cb >= volume_cb) return;
    constexpr double k = 0.70710678118654752440;
    constexpr int s1[4] = {1, 2, 3, 0}, s2[4] = {3, 0, 1, 2};
    if constexpr (to_native) {
      constexpr double K1[4] = {k, -k, -k, -k}, K2[4] = {k, -k, k, k};
      real v[24];
#pragma unroll
      for (int s = 0; s < 4; s++)
#pragma unroll
        for (int c = 0; c < 6; c++)
          v[s * 6 + c] = (real)(K1[s] * (double)host[(size_t)x_cb * 24 + s1[s] * 6 + c] + K2[s] * (double)host[(size_t)x_cb * 24 + s2[s] * 6 + c]);
      nat.save(v, x_cb);
    } else {
      constexpr double K1[4] = {-k, k, k, k}, K2[4] = {-k, k, -k, -k};
      real v[24];
      nat.template load<Cache::STREAM>(v, x_cb);
#pragma unroll
      for (int s = 0; s < 4; s++)
#pragma unroll
        for (int c = 0; c < 6; c++)
          host[(size_t)x_cb * 24 + s * 6 + c] = (H)(K1[s] * (double)v[s1[s] * 6 + c] + K2[s] * (double)v[s2[s] * 6 + c]);
    }
  }

  template <class P> int launch_copy_precision(const CopyRequest &rq)
  {
    SpinorView<P> nat;
    fill_spinor(nat, rq.native, rq.native_norm, rq.volume_cb);
    const int blocks = (rq.volume_cb + 127) / 128;
    cudaStream_t s = (cudaStream_t)rq.stream;
    if (rq.host_precision == 8) {
      if (rq.to_native)
        copy_spinor_kernel<P, double, true><<<blocks, 128, 0, s>>>(nat, (double *)rq.host, rq.volume_cb);
      else
        copy_spinor_kernel<P, double, false><<<blocks, 128, 0, s>>>(nat, (double *)rq.host, rq.volume_cb);
    } else {
      if (rq.to_native)
        copy_spinor_kernel<P, float, true><<<blocks, 128, 0, s>>>(nat, (float *)rq.host, rq.volume_cb);
      else
        copy_spinor_kernel<P, float, false><<<blocks, 128, 0, s>>>(nat, (float *)rq.host, rq.volume_cb);
    }
    count_launch();
    return check_cuda(cudaGetLastError(), "copy_spinor launch");
  }

  // ---- gauge: QDP host order -> native packed order incl. the ghost links in the pad (loadGaugeQuda's device work)
  template <class P, int recon, typename H> struct GaugeCopyArgs {
    Geom geom;
    typename P::store *g[2];
    int stride;
    const H *qdp[4];
    const H *ghost[4];
    typename P::real link_max_inv;
  };

  template <class P, int recon, typename H>
  __global__ void __launch_bounds__(128) copy_gauge_kernel(const __grid_constant__ GaugeCopyArgs<P, recon, H> arg)
  {
    using real = typename P::real;
    using store = typename P::store;
    constexpr int N = GaugeVec<P, recon>::N;
    const Geom &g = arg.geom;
    const int mu = blockIdx.y >> 1, parity = blockIdx.y & 1;
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= g.volume_cb + g.face_cb[mu]) return;
    const H *src;
    if (idx < g.volume_cb) {
      src = arg.qdp[mu] + ((size_t)parity * g.volume_cb + idx) * 18;
    } else {
      const int f = idx - g.volume_cb;
      if (arg.ghost[mu]) {
        src = arg.ghost[mu] + ((size_t)parity * g.face_cb[mu] + f) * 18;
      } else { // this rank is its own backward neighbour: links of the x[mu] = X[mu]-1 slice, in face order
        int x[4];
        coords_from_face(x, g, mu, g.X[mu] - 1, f, parity);
        src = arg.qdp[mu] + ((size_t)parity * g.volume_cb + cb_from_coords(x, g)) * 18;
      }
    }
    double u[18];
#pragma unroll
    for (int i = 0; i < 18; i++) u[i] = (double)src[i];
    real t[recon];
    if constexpr (recon == 18) {
#pragma unroll
      for (int i = 0; i < 18; i++) t[i] = (real)(P::fixed ? u[i] * (double)arg.link_max_inv : u[i]);
    } else if constexpr (recon == 12) {
#pragma unroll
      for (int i = 0; i < 12; i++) t[i] = (real)u[i];
    } else { // gauge_field_order.h:1303-1316
      constexpr double inv_pi = 0.31830988618379067154;
      t[0] = (real)(atan2(u[7], u[6]) * inv_pi);
      t[1] = (real)(atan2(-u[13], -u[12]) * inv_pi);
      t[2] = (real)u[8];
      t[3] = (real)u[9];
      t[4] = (real)u[10];
      t[5] = (real)u[11];
      t[6] = (real)u[0];
      t[7] = (real)u[1];
    }
#pragma unroll
    for (int i = 0; i < recon; i++) {
      store v;
      if constexpr (P::fixed)
        v = f2s((float)t[i] * kFixedMax);
      else
        v = t[i];
      arg.g[parity][((size_t)(mu * (recon / N) + i / N) * arg.stride + idx) * N + i % N] = v;
    }
  }

  template <class P, int recon, typename H> int launch_gauge_copy_typed(const GaugeCopyRequest &rq)
  {
    GaugeCopyArgs<P, recon, H> a;
    geom_init(a.geom, rq.X);
    a.g[0] = reinterpret_cast<typename P::store *>(const_cast<void *>(rq.native.gauge));
    a.g[1] = reinterpret_cast<typename P::store *>(reinterpret_cast<char *>(const_cast<void *>(rq.native.gauge)) + rq.native.parity_stride_bytes);
    a.stride = rq.native.stride;
    a.link_max_inv = (typename P::real)(1.0 / rq.native.link_max);
    int max_face = 0;
    for (int d = 0; d < 4; d++) {
      a.qdp[d] = reinterpret_cast<const H *>(rq.qdp[d]);
      a.ghost[d] = reinterpret_cast<const H *>(rq.ghost[d]);
      if (a.geom.face_cb[d] > max_face) max_face = a.geom.face_cb[d];
    }
    if (a.stride < a.geom.volume_cb + max_face) return set_error(B200_ERR_INVALID, "gauge stride %d leaves no room for the ghost pad", a.stride);
    dim3 grid((a.geom.volume_cb + max_face + 127) / 128, 8, 1);
    copy_gauge_kernel<P, recon, H><<<grid, 128, 0, (cudaStream_t)rq.stream>>>(a);
    count_launch();
    return check_cuda(cudaGetLastError(), "copy_gauge launch");
  }

  template <class P> int launch_gauge_copy_precision(const GaugeCopyRequest &rq)
  {
    const bool dbl = rq.host_precision == 8;
    switch (rq.native.reconstruct) {
    case 18: return dbl ? launch_gauge_copy_typed<P, 18, double>(rq) : launch_gauge_copy_typed<P, 18, float>(rq);
    case 12: return dbl ? launch_gauge_copy_typed<P, 12, double>(rq) : launch_gauge_copy_typed<P, 12, float>(rq);
    case 8: return dbl ? launch_gauge_copy_typed<P, 8, double>(rq) : launch_gauge_copy_typed<P, 8, float>(rq);
    }
    return set_error(B200_ERR_INVALID, "reconstruct %d not in {18,12,8}", rq.native.reconstruct);
  }

  // ---- clover: packed host order -> native (A/2, optional 28-real compression, block-float scale)
  template <class P, typename H>
  __global__ void __launch_bounds__(128) copy_clover_kernel(typename P::store *c0, typename P::store *c1, const H *packed,
                                                            int volume_cb, int compressed, double diagonal, double nrm_inv)
  {
    using store = typename P::store;
    constexpr int N = P::Ns;
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    if (x >= volume_cb) return;
    const int parity = blockIdx.y;
    store *dst = parity ? c1 : c0;
    const H *src = packed + ((size_t)parity * volume_cb + x) * 72;
    const int CB = compressed ? 28 : 36;
#pragma unroll
    for (int chi = 0; chi < 2; chi++) {
      double a[36];
#pragma unroll
      for (int i = 0; i < 36; i++) a[i] = 0.5 * (double)src[chi * 36 + i];
      for (int k = 0; k < CB; k++) {
        double v;
        if (!compressed)
          v = a[k];
        else if (k < 3)
          v = a[k] - diagonal;
        else if (k == 3)
          v = 0.0;
        else
          v = a[k + 2];
        const int flat = chi * CB + k;
        store o;
        if constexpr (P::fixed)
          o = f2s((float)(v * nrm_inv));
        else
          o = (store)v;
        dst[((size_t)(flat / N) * volume_cb + x) * N + flat % N] = o;
      }
    }
  }

  template <class P> int launch_clover_copy_precision(const CloverCopyRequest &rq)
  {
    Geom g;
    geom_init(g, rq.X);
    auto *c0 = reinterpret_cast<typename P::store *>(const_cast<void *>(rq.native.clover));
    auto *c1 = reinterpret_cast<typename P::store *>(reinterpret_cast<char *>(const_cast<void *>(rq.native.clover)) + rq.native.parity_stride_bytes);
    const double nrm_inv = P::fixed ? (2.0 * 32767.0) / rq.native.max_element : 1.0;
    dim3 grid((g.volume_cb + 127) / 128, 2, 1);
    cudaStream_t s = (cudaStream_t)rq.stream;
    if (rq.host_precision == 8)
      copy_clover_kernel<P, double><<<grid, 128, 0, s>>>(c0, c1, (const double *)rq.packed, g.volume_cb, rq.native.compressed, rq.native.diagonal, nrm_inv);
    else
      copy_clover_kernel<P, float><<<grid, 128, 0, s>>>(c0, c1, (const float *)rq.packed, g.volume_cb, rq.native.compressed, rq.native.diagonal, nrm_inv);
    count_launch();
    return check_cuda(cudaGetLastError(), "copy_clover launch");
  }

  // ------------------------------------------------------------------ host side: issue the launch plan of one request
  template <class P, int recon, bool dagger, bool xpay, OpType op>
  int launch_config(OpCfg<dagger, xpay, op>, const LaunchRequest &rq, const DslashArgs<P, recon> &arg)
  {
    LaunchPlan pl;
    if (int rc = plan_dslash(pl, rq, arg)) return rc;
    cudaStream_t s = (cudaStream_t)rq.stream;
    for (int i = 0; i < pl.n; i++) {
      const LaunchStep &l = pl.step[i];
      const dim3 grid(l.grid[0], l.grid[1], l.grid[2]);
      if (l.kind == LAUNCH_INTERIOR && !l.masked) {
        dslash_interior_kernel<P, recon, dagger, xpay, op, false><<<grid, l.threads, 0, s>>>(arg, l.tm);
      } else if constexpr (!has_partitioned_kernels(op)) {
        return refuse_partitioned_tm_pc_pre();
      } else {
        switch (l.kind) {
        case LAUNCH_INTERIOR: dslash_interior_kernel<P, recon, dagger, xpay, op, true><<<grid, l.threads, 0, s>>>(arg, l.tm); break;
        case LAUNCH_BOUNDARY: dslash_boundary_kernel<P, recon, dagger, xpay, op><<<grid, l.threads, 0, s>>>(arg, l.tm, l.st); break;
        case LAUNCH_EXTERIOR: dslash_exterior_kernel<P, recon, dagger, xpay, op><<<grid, l.threads, 0, s>>>(arg); break;
        case LAUNCH_FUSED: {
          PackArgs<P> pk {};
          if (rq.fused_pack) fill_pack_args(pk, *rq.fused_pack);
          dslash_fused_kernel<P, recon, dagger, xpay, op><<<grid, l.threads, 0, s>>>(arg, l.tm, pk, l.fs);
          break;
        }
        }
      }
      count_launch();
    }
    return check_cuda(cudaGetLastError(), rq.fused_pack ? "fused dslash launch" : "dslash launch");
  }

  template <class P> int launch_precision(const LaunchRequest &rq)
  {
    return dispatch_dslash<P>(rq, [&](auto c, const auto &arg) { return launch_config(c, rq, arg); });
  }

  template <class P> int launch_clover_precision(const CloverRequest &rq)
  {
    SpinorView<P> out, in;
    CloverView<P> A;
    fill_spinor(out, rq.out, rq.out_norm, rq.volume_cb);
    fill_spinor(in, rq.in, rq.in_norm, rq.volume_cb);
    fill_clover(A, rq.A, rq.volume_cb);
    const int blocks = (rq.volume_cb + 127) / 128;
    cudaStream_t s = (cudaStream_t)rq.stream;
    if (rq.inverse)
      clover_apply_kernel<P, true><<<blocks, 128, 0, s>>>(out, in, A, rq.volume_cb, rq.parity);
    else
      clover_apply_kernel<P, false><<<blocks, 128, 0, s>>>(out, in, A, rq.volume_cb, rq.parity);
    count_launch();
    return check_cuda(cudaGetLastError(), "clover launch");
  }

  template <class P> int launch_twist_precision(const TwistRequest &rq)
  {
    SpinorView<P> out, in;
    fill_spinor(out, rq.out, rq.out_norm, rq.volume_cb);
    fill_spinor(in, rq.in, rq.in_norm, rq.volume_cb);
    twist_gamma5_kernel<P><<<(rq.volume_cb + 255) / 256, 256, 0, (cudaStream_t)rq.stream>>>(out, in, rq.volume_cb, (typename P::real)rq.a,
                                                                                          (typename P::real)rq.b);
    count_launch();
    return check_cuda(cudaGetLastError(), "twist launch");
  }

  template <class P> int launch_pack_precision(const PackRequest &rq)
  {
    int gx;
    if (int rc = pack_blocks(gx, rq)) return rc;
    if (!gx) return 0;
    PackArgs<P> arg;
    fill_pack_args(arg, rq);
    pack_kernel<P><<<dim3(gx, 8, 1), 128, 0, (cudaStream_t)rq.stream>>>(arg);
    count_launch();
    return check_cuda(cudaGetLastError(), "pack launch");
  }

  template <class P> int launch_pack_multi_precision(const PackRequest &rq, const PackBatchRequest &b)
  {
    int gx;
    if (int rc = pack_blocks(gx, rq)) return rc;
    if (!gx) return 0;
    PackArgs<P> arg;
    fill_pack_args(arg, rq);
    PackBatch<P> batch;
    fill_pack_batch(batch, b, arg.geom.volume_cb);
    pack_multi_kernel<P><<<dim3(gx, 8, b.n_src), 128, 0, (cudaStream_t)rq.stream>>>(arg, batch);
    count_launch();
    return check_cuda(cudaGetLastError(), "batched pack launch");
  }

} // namespace b200
