// CUDA side of the TMA-staged marching kernel (plan + site arithmetic: tma.h): mbarrier pipeline, cp.async.bulk.tensor
// box loads issued by a producer warp, consumer warps doing LDS + FFMA only, tensor-map encoding on the host.
#pragma once

#include <cuda.h>
#include <cuda_runtime.h>

#include "plan.h"
#include "tma.h"

namespace b200
{

  struct alignas(64) TmaMaps {
    CUtensorMap m[2][TM_COUNT]; // [output parity (0 if single parity)][shape]
  };

  // ---- mbarrier / TMA primitives (PTX ISA 8.x: mbarrier, cp.async.bulk.tensor) --------------------------------------
  __device__ __forceinline__ void mbar_init(unsigned bar, unsigned count)
  {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
  }
  __device__ __forceinline__ void mbar_expect_tx(unsigned bar, unsigned bytes)
  {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
  }
  __device__ __forceinline__ void mbar_arrive(unsigned bar)
  {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
  }
  __device__ __forceinline__ bool mbar_try(unsigned bar, unsigned parity)
  {
    unsigned ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok)
                 : "r"(bar), "r"(parity)
                 : "memory");
    return ok != 0;
  }
  // Wait for the phase with parity `parity` to complete.  A pipeline bug must never hang the GPU: after 2^26 failed
  // probes (each try_wait suspends the thread for a while, so this is seconds) the kernel traps -- the launch fails with
  // an error instead of spinning until the watchdog.
  __device__ __forceinline__ void mbar_wait(unsigned bar, unsigned parity)
  {
    if (mbar_try(bar, parity)) return;
    int spins = 0;
    while (!mbar_try(bar, parity)) {
      if (++spins > (1 << 26)) __trap();
    }
  }

  // one lane of a converged warp (elect.sync): ptxas knows that exactly one thread executes the guarded code, which lets
  // it issue uniform-datapath instructions (UTMALDG, SYNCS) there without a per-lane serialisation loop
  __device__ __forceinline__ bool elect_one()
  {
    unsigned pred = 0;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
  }

  __device__ __forceinline__ unsigned long long l2_policy_evict_first()
  {
    unsigned long long pol;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
    return pol;
  }
  __device__ __forceinline__ unsigned long long l2_policy_evict_last()
  {
    unsigned long long pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
  }

  // one box load global -> shared, completion counted in bytes on `bar`
  __device__ __forceinline__ void tma_load_box(unsigned dst, const CUtensorMap *map, unsigned bar, const int *c, unsigned long long policy)
  {
    asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint"
                 " [%0], [%1, {%2, %3, %4, %5, %6}], [%7], %8;" ::"r"(dst),
                 "l"(map), "r"(c[0]), "r"(c[1]), "r"(c[2]), "r"(c[3]), "r"(c[4]), "r"(bar), "l"(policy)
                 : "memory");
  }

  // pull one box into L2 only (no shared memory, no completion tracking)
  __device__ __forceinline__ void tma_prefetch_box(const CUtensorMap *map, const int *c)
  {
    asm volatile("cp.async.bulk.prefetch.tensor.5d.L2.global.tile [%0, {%1, %2, %3, %4, %5}];" ::"l"(map), "r"(c[0]), "r"(c[1]),
                 "r"(c[2]), "r"(c[3]), "r"(c[4])
                 : "memory");
  }

  template <class P, int recon, bool dagger, bool xpay, OpType op, int PD>
  __global__ void __launch_bounds__(kTmaMaxConsumers + 32, 1)
    dslash_tma_kernel(const __grid_constant__ DslashArgs<P, recon> arg, const __grid_constant__ TmaPlan plan,
                      const __grid_constant__ TmaMaps maps)
  {
    using real = typename P::real;
    using Raw = typename GaugeView<P, recon>::Raw;
    constexpr bool LSTREAM = PD > 0; // PD: prefetch distance of the register-stream links (0: links via shared memory)
    extern __shared__ __align__(1024) unsigned char tma_smem[];
    const unsigned sbase = (unsigned)__cvta_generic_to_shared(tma_smem);
    const unsigned bars = sbase + plan.off_bar;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int NCS = plan.n_center_slots, NHS = plan.n_halo_slots, NL = plan.n_link_slots;

    if (tid == 0) {
      for (int s = 0; s < kTmaMaxCenterSlots; s++) {
        mbar_init(bars + 8 * tma_bar_full_c(s), 1);
        mbar_init(bars + 8 * tma_bar_empty_c(s), plan.n_cwarps);
      }
      for (int s = 0; s < kTmaMaxHaloSlots; s++) {
        mbar_init(bars + 8 * tma_bar_full_h(s), 1);
        mbar_init(bars + 8 * tma_bar_empty_h(s), plan.n_cwarps);
      }
      for (int s = 0; s < kTmaMaxLinkSlots; s++) {
        mbar_init(bars + 8 * tma_bar_full_l(s), 1);
        mbar_init(bars + 8 * tma_bar_empty_l(s), plan.n_cwarps);
      }
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    int w0, w1;
    tma_work_range(w0, w1, plan, blockIdx.x, gridDim.x);
    if (w0 >= w1) return;

    if (warp == plan.n_cwarps) {
      // ================================================================== producer: one thread issues every box load
      // The whole warp runs the (warp-uniform) program so that its address arithmetic stays on the uniform datapath; only
      // lane 0 touches the mbarriers' transaction counts and issues the TMA instructions.
      struct Issuer {
        const TmaPlan &plan;
        const TmaMaps &maps;
        unsigned sbase, bars, center_tx, halo_tx, link_tx;
        unsigned long long pol_links, pol_spinor;
        bool leader;
        TmaPos cp, hp, lp; // ring positions of the next centre / halo / link load (loads are requested in sequence)
        int cn, hn;
        long long ln;
        __device__ __forceinline__ const CUtensorMap *map(const TmaItem &it, int id) const
        {
          return &maps.m[plan.n_parity == 2 ? it.par : 0][id];
        }
        __device__ __forceinline__ void center(int n, const TmaItem &it, int slice)
        {
          if (n != cn) __trap(); // the program requests centre loads in sequence
          if (n >= plan.n_center_slots) mbar_wait(bars + 8 * tma_bar_empty_c(cp.slot), cp.phase ^ 1u);
          const unsigned full = bars + 8 * tma_bar_full_c(cp.slot);
          TmaBox b;
          tma_center_box(b, it, slice);
          if (elect_one()) {
            mbar_expect_tx(full, center_tx);
            tma_load_box(sbase + plan.off_center + cp.slot * plan.center_bytes + b.dst, map(it, b.map), full, b.c, pol_spinor);
          }
          cp = tma_pos_next(cp, plan.n_center_slots);
          cn++;
        }
        __device__ __forceinline__ void halo(int n, const TmaItem &it)
        {
          if (n != hn) __trap();
          if (n >= plan.n_halo_slots) mbar_wait(bars + 8 * tma_bar_empty_h(hp.slot), hp.phase ^ 1u);
          const unsigned full = bars + 8 * tma_bar_full_h(hp.slot);
          TmaBox b[4];
          tma_halo_boxes(b, plan, it);
          if (elect_one()) {
            mbar_expect_tx(full, halo_tx);
#pragma unroll
            for (int k = 0; k < 4; k++)
              tma_load_box(sbase + plan.off_halo + hp.slot * plan.halo_bytes + b[k].dst, map(it, b[k].map), full, b[k].c, pol_spinor);
          }
          hp = tma_pos_next(hp, plan.n_halo_slots);
          hn++;
        }
        __device__ __forceinline__ void prefetch_link(const TmaItem &it, int d)
        {
          TmaBox b[3];
          const int nb = tma_link_boxes(b, plan, it, d);
          if (elect_one())
            for (int k = 0; k < nb; k++) tma_prefetch_box(map(it, b[k].map), b[k].c);
        }
        __device__ __forceinline__ void link(long long n, const TmaItem &it, int d)
        {
          if (n != ln) __trap();
          if (n >= plan.n_link_slots) mbar_wait(bars + 8 * tma_bar_empty_l(lp.slot), lp.phase ^ 1u);
          const unsigned full = bars + 8 * tma_bar_full_l(lp.slot);
          TmaBox b[3];
          const int nb = tma_link_boxes(b, plan, it, d);
          if (elect_one()) {
            mbar_expect_tx(full, link_tx);
            for (int k = 0; k < nb; k++)
              tma_load_box(sbase + plan.off_link + lp.slot * plan.link_bytes + b[k].dst, map(it, b[k].map), full, b[k].c, pol_links);
          }
          lp = tma_pos_next(lp, plan.n_link_slots);
          ln++;
        }
      };
      Issuer is {plan, maps, sbase, bars, (unsigned)(plan.NC * plan.srow), (unsigned)(plan.NH * plan.srow),
                 (unsigned)(2 * plan.NC * plan.grow), l2_policy_evict_first(), l2_policy_evict_last(), lane == 0,
                 TmaPos {0, 0}, TmaPos {0, 0}, TmaPos {0, 0}, 0, 0, 0};
      tma_producer_program(plan, w0, w1, is);
      return;
    }

    // ==================================================================== consumers: one thread per site of the tile
    TmaThread th;
    tma_thread_init(th, plan, tid);
    TmaPos c0p {0, 0}; // ring position of the centre load holding slice t-1 of the current item
    TmaPos hp {0, 0}, lp {0, 0};
    TmaItem it;
    tma_item(it, plan, w0);
    TmaSite cur;
    tma_site(cur, plan, th, it);
    Raw lk[LSTREAM ? 8 : 1];
    if constexpr (LSTREAM) {
      if (th.active) tma_load_links<P, recon, PD>(lk, arg.U, cur);
    }
    for (int w = w0; w < w1; w++) {
      const bool first = (w == w0) || (it.t == 0);
      const bool last = (w == w1 - 1) || (it.t == plan.T - 1);
      const bool have_next = w + 1 < w1;
      TmaItem nit = it;
      TmaSite nxt = cur;
      if (have_next) {
        tma_item_next(nit, it, plan, w + 1);
        tma_site(nxt, plan, th, nit);
      }
      const TmaPos c1p = tma_pos_next(c0p, NCS), c2p = tma_pos_next(c1p, NCS);
      if (first) {
        mbar_wait(bars + 8 * tma_bar_full_c(c0p.slot), c0p.phase);
        mbar_wait(bars + 8 * tma_bar_full_c(c1p.slot), c1p.phase);
      }
      mbar_wait(bars + 8 * tma_bar_full_c(c2p.slot), c2p.phase);
      mbar_wait(bars + 8 * tma_bar_full_h(hp.slot), hp.phase);
      TmaBases b;
      b.cm = sbase + plan.off_center + c0p.slot * plan.center_bytes;
      b.c0 = sbase + plan.off_center + c1p.slot * plan.center_bytes;
      b.cp = sbase + plan.off_center + c2p.slot * plan.center_bytes;
      b.halo = sbase + plan.off_halo + hp.slot * plan.halo_bytes;
      real acc[24];
#pragma unroll
      for (int i = 0; i < 24; i++) acc[i] = 0;

      if constexpr (LSTREAM) {
        if (th.active) {
          tma_hop_pair_stream<P, recon, dagger, 0, PD>(acc, arg.U, lk, plan, th, b, cur, nxt, have_next);
          tma_hop_pair_stream<P, recon, dagger, 1, PD>(acc, arg.U, lk, plan, th, b, cur, nxt, have_next);
          tma_hop_pair_stream<P, recon, dagger, 2, PD>(acc, arg.U, lk, plan, th, b, cur, nxt, have_next);
          tma_hop_pair_stream<P, recon, dagger, 3, PD>(acc, arg.U, lk, plan, th, b, cur, nxt, have_next);
        }
        __syncwarp();
      } else {
#define B2_TMA_DIM(D)                                                                                                  \
  {                                                                                                                    \
    mbar_wait(bars + 8 * tma_bar_full_l(lp.slot), lp.phase);                                                           \
    const unsigned stage = sbase + plan.off_link + lp.slot * plan.link_bytes;                                          \
    if (th.active) tma_hop_pair<P, recon, dagger, D>(acc, arg.U, plan, th, b, stage, cur);                             \
    __syncwarp();                                                                                                      \
    if (lane == 0) mbar_arrive(bars + 8 * tma_bar_empty_l(lp.slot));                                                   \
    lp = tma_pos_next(lp, NL);                                                                                         \
  }
        B2_TMA_DIM(0)
        B2_TMA_DIM(1)
        B2_TMA_DIM(2)
        B2_TMA_DIM(3)
#undef B2_TMA_DIM
      }
      // every shared-memory operand of this item has been read: hand the oldest slice and the halo rows back
      if (lane == 0) {
        mbar_arrive(bars + 8 * tma_bar_empty_c(c0p.slot));
        mbar_arrive(bars + 8 * tma_bar_empty_h(hp.slot));
        if (last) {
          mbar_arrive(bars + 8 * tma_bar_empty_c(c1p.slot));
          mbar_arrive(bars + 8 * tma_bar_empty_c(c2p.slot));
        }
      }
      if (th.active) tma_epilogue<P, recon, dagger, xpay, op>(acc, arg, cur.x_cb, cur.par);
      c0p = last ? tma_pos_next(c2p, NCS) : c1p;
      hp = tma_pos_next(hp, NHS);
      it = nit;
      cur = nxt;
    }
  }

  // ---- host: tensor-map encoding + launch -------------------------------------------------------------------------
  typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                    const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

  inline EncodeTiledFn tma_encode_fn()
  {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
      tried = true;
      void *p = nullptr;
      cudaDriverEntryPointQueryResult q;
      if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
        fn = reinterpret_cast<EncodeTiledFn>(p);
      else
        cudaGetLastError();
    }
    return fn;
  }

  inline int tma_encode(CUtensorMap &m, const TmaDesc &d)
  {
    EncodeTiledFn fn = tma_encode_fn();
    if (!fn) return set_error(B200_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
    cuuint64_t dim[5], stride[4];
    cuuint32_t box[5], es[5] = {1, 1, 1, 1, 1};
    for (int i = 0; i < 5; i++) dim[i] = d.dim[i], box[i] = d.box[i];
    for (int i = 0; i < 4; i++) stride[i] = d.stride[i + 1];
    const CUresult r = fn(&m, CU_TENSOR_MAP_DATA_TYPE_UINT32, 5, const_cast<void *>(d.base), dim, stride, box, es,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return set_error(B200_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
    return 0;
  }

  inline int tma_sm_count()
  {
    static int n = 0;
    if (!n) {
      int dev = 0;
      cudaGetDevice(&dev);
      if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    }
    return n;
  }

  template <class P, int recon, bool dagger, bool xpay, OpType op>
  int launch_tma(OpCfg<dagger, xpay, op>, const LaunchRequest &rq, const DslashArgs<P, recon> &arg)
  {
    TmaPlan plan;
    TmaKnobs knobs {rq.tma_ty, rq.tma_tz, rq.tma_link_slots, rq.tma_center_slots, rq.tma_halo_slots, rq.tma_l2_prefetch};
    if (!tma_make_plan<P, recon>(plan, arg.geom, arg.n_parity, arg.parity, knobs)) return kTmaSkip;
    TmaMaps maps;
    memset(&maps, 0, sizeof(maps));
    for (int pi = 0; pi < arg.n_parity; pi++) {
      TmaDesc d[TM_COUNT];
      tma_make_descs(d, arg, plan, arg.n_parity == 2 ? pi : arg.parity);
      for (int k = 0; k < TM_COUNT; k++) {
        if (!d[k].valid) continue;
        if (!tma_desc_ok(d[k])) return kTmaSkip;
        if (int rc = tma_encode(maps.m[pi][k], d[k])) return rc;
      }
    }
    const int grid = tma_grid(rq, plan.n_items, tma_sm_count());
    const int threads = (plan.n_cwarps + 1) * 32;
    cudaStream_t s = (cudaStream_t)rq.stream;
    auto go = [&](auto kern) -> int {
      if (int rc = check_cuda(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kTmaSmemBudget), "TMA kernel smem attribute"))
        return rc;
      kern<<<grid, threads, plan.smem_bytes, s>>>(arg, plan, maps);
      return 0;
    };
    int rc = 0;
    if (plan.n_link_slots > 0)
      rc = go(dslash_tma_kernel<P, recon, dagger, xpay, op, 0>);
    else if (rq.tma_prefetch == 2)
      rc = go(dslash_tma_kernel<P, recon, dagger, xpay, op, 2>);
    else if (rq.tma_prefetch == 4)
      rc = go(dslash_tma_kernel<P, recon, dagger, xpay, op, 4>);
    else
      rc = go(dslash_tma_kernel<P, recon, dagger, xpay, op, 3>);
    if (rc) return rc;
    count_launch();
    return check_cuda(cudaGetLastError(), "dslash TMA launch");
  }

  template <class P> int launch_tma_precision(const LaunchRequest &rq)
  {
    return dispatch_tma<P>(rq, [&](auto c, const auto &arg) { return launch_tma(c, rq, arg); });
  }

} // namespace b200
