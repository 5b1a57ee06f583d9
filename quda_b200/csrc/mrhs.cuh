// Multi-RHS (batched) Dslash: kernel wrappers + the per-precision launcher that issues plan.h's multi-RHS schedule.  The site code is dslash_site_mrhs
// (dslash_site.h); one translation unit per storage precision includes this header (inst_mrhs_*.cu).
//
// Reference interface: the cvector_ref<ColorSpinorField> form of ApplyWilson / ApplyWilsonClover /
// ApplyWilsonCloverPreconditioned (include/dslash_quda.h:83-234), i.e. WilsonArg::out/in/x[MAX_MULTI_RHS] and the
// source index in the thread grid (include/kernels/dslash_wilson.cuh:37-69).
#pragma once

#include <cuda_runtime.h>

#include "dslash_site.h"
#include "plan.h"

namespace b200
{

  // Register budget: NS accumulators of 24 reals + the NS x 24-real spinor loads in flight.  2 CTAs of <= 128 threads
  // per SM gives ptxas the full 255 registers (fp64 NS = 2, fp32/half NS = 4); NS = 2 in fp32/half fits 168.
#ifndef B2_MRHS_MINBLOCKS_4
#define B2_MRHS_MINBLOCKS_4 2
#endif
#ifndef B2_MRHS_MINBLOCKS_2
#define B2_MRHS_MINBLOCKS_2 3
#endif
  template <class P, int NS> struct MrhsMinBlocks { static constexpr int value = NS >= 4 ? B2_MRHS_MINBLOCKS_4 : B2_MRHS_MINBLOCKS_2; };
  template <int NS> struct MrhsMinBlocks<PrecF64, NS> { static constexpr int value = 2; };

  template <class P, int recon, bool dagger, bool xpay, OpType op, int NS>
  __global__ void __launch_bounds__(B2_MAXTILE, MrhsMinBlocks<P, NS>::value)
    dslash_mrhs_kernel(const __grid_constant__ DslashArgs<P, recon> arg, const __grid_constant__ MrhsFields<P, NS> f,
                       const __grid_constant__ TileMap tm)
  {
    int x[4], x_cb, parity;
    if (!tile_site(x, x_cb, parity, arg.geom, tm, arg.n_parity, arg.parity, blockIdx.x, blockIdx.y, blockIdx.z, threadIdx.x))
      return;
    dslash_site_mrhs<P, recon, dagger, xpay, op, NS>(arg, f, x, x_cb, parity);
  }

  // ---- CTA flavour: blockDim = (tile sites, sources per CTA); blockIdx.x = tile * n_batch + batch, so the CTAs that
  // share a tile's links are adjacent in launch order (L2 serves what L1 cannot)
  // Occupancy / register configurations of the CTA flavour (B200_MRHS_CTA_CFG): with the links shared through L1 / L2
  // the DRAM stream has head-room, so the kernel is bound by the per-thread load-latency chain and more resident warps
  // (fewer registers, no register-resident link preload) can pay:  cfg 0 = the single-source budget (128 regs, links
  // preloaded), cfg 1 = 6 CTAs of 128 threads (85 regs), cfg 2 = 8 CTAs (64 regs); fp64: 255 / 168 / 128 regs.
  template <class P, int CFG> struct MrhsCtaCfg {
    static constexpr int min_blocks = CFG == 0 ? 4 : (CFG == 1 ? 6 : 8);
    static constexpr bool preload = CFG == 0;
  };
  template <int CFG> struct MrhsCtaCfg<PrecF64, CFG> {
    static constexpr int min_blocks = CFG == 0 ? 2 : (CFG == 1 ? 3 : 4);
    static constexpr bool preload = false;
  };

  template <class P, int recon, bool dagger, bool xpay, OpType op, bool l1_links, int CFG>
  __global__ void __launch_bounds__(B2_MAXTILE, MrhsCtaCfg<P, CFG>::min_blocks)
    dslash_mrhs_cta_kernel(const __grid_constant__ DslashArgs<P, recon> arg, const __grid_constant__ MrhsViews<P> f,
                           const __grid_constant__ TileMap tm, int n_src, int n_batch)
  {
    const unsigned tile = blockIdx.x / (unsigned)n_batch;
    const int s = (int)(blockIdx.x - tile * n_batch) * blockDim.y + threadIdx.y;
    if (s >= n_src) return;
    int x[4], x_cb, parity;
    if (!tile_site(x, x_cb, parity, arg.geom, tm, arg.n_parity, arg.parity, tile, blockIdx.y, blockIdx.z, threadIdx.x)) return;
    dslash_site_src<P, recon, dagger, xpay, op, l1_links ? Cache::REUSE : Cache::STREAM, MrhsCtaCfg<P, CFG>::preload>(
      arg, f.in[s][1 - parity], f.out[s][parity], f.x[s][parity], x, x_cb, parity);
  }

  template <class P, int recon, bool dagger, bool xpay, OpType op>
  int launch_mrhs_cta(OpCfg<dagger, xpay, op>, const MrhsRequest &rq, const DslashArgs<P, recon> &arg)
  {
    MrhsViews<P> f;
    fill_mrhs_views(f, rq);
    MrhsGrid m;
    if (int rc = plan_mrhs(m, rq, arg, true)) return rc;
    if (!m.gx) return 0;
    const dim3 grid(m.gx * m.n_batch, m.gy, m.gz), block(m.threads, m.nsb, 1);
    cudaStream_t st = (cudaStream_t)rq.base.stream;
#define B2_CTA_LAUNCH(L1, CFG) \
  dslash_mrhs_cta_kernel<P, recon, dagger, xpay, op, L1, CFG><<<grid, block, 0, st>>>(arg, f, m.tm, rq.n_src, m.n_batch)
    if (!rq.l1_links)
      B2_CTA_LAUNCH(false, 0);
    else if (rq.cta_cfg == 1)
      B2_CTA_LAUNCH(true, 1);
    else if (rq.cta_cfg == 2)
      B2_CTA_LAUNCH(true, 2);
    else
      B2_CTA_LAUNCH(true, 0);
#undef B2_CTA_LAUNCH
    count_launch();
    return check_cuda(cudaGetLastError(), "multi-RHS (CTA) dslash launch");
  }

  template <int NS, class P, int recon, bool dagger, bool xpay, OpType op>
  int launch_mrhs_batch(OpCfg<dagger, xpay, op>, const MrhsRequest &rq, const DslashArgs<P, recon> &arg, int s0)
  {
    MrhsFields<P, NS> f;
    fill_mrhs_fields(f, rq, s0);
    MrhsGrid m;
    if (int rc = plan_mrhs(m, rq, arg, false)) return rc;
    if (!m.gx) return 0;
    dslash_mrhs_kernel<P, recon, dagger, xpay, op, NS><<<dim3(m.gx, m.gy, m.gz), m.threads, 0, (cudaStream_t)rq.base.stream>>>(arg, f, m.tm);
    count_launch();
    return check_cuda(cudaGetLastError(), "multi-RHS dslash launch");
  }

  template <class P> int launch_mrhs_precision(const MrhsRequest &rq)
  {
    return dispatch_mrhs<P>(rq, [&](auto c, const auto &arg, auto ns, int s0) -> int {
      constexpr int NS = decltype(ns)::value;
      if constexpr (NS == 0)
        return launch_mrhs_cta(c, rq, arg);
      else if constexpr (NS == 1) // the odd one out: the single-source kernel (inst_*.cu)
        return launch_precision<P>(mrhs_source(rq, s0));
      else
        return launch_mrhs_batch<NS>(c, rq, arg, s0);
    });
  }

} // namespace b200
