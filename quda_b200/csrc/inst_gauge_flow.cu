// Kernels of b200_gauge_flow and b200_gauge_observables (site code: gauge_flow.h).  The flow runs one launch per RK3 stage,
// one thread per (site, direction, parity) link, ping-ponging between the output and one scratch link field; the
// observables run one thread per site and reduce in inst_gauge.cu's two fixed-order stages, so repeated calls give
// bit-identical results.
#include "gauge_flow.h"

namespace b200
{

  // inst_clover_build.cu: out[g] = fixed-order sum of the n partials of group g = blockIdx.x (one CTA per group)
  __global__ void clover_trlog_kernel(const double *partial, int n, double *trlog);
  // inst_gauge.cu: the second stage of the sums, the copy of the `groups` sums to g, then scratch freed and the stream synchronised
  int finish_sums(double *scratch, int nblk, int groups, double *g, cudaStream_t s);

  template <typename T> __global__ void __launch_bounds__(kGaugeThreads) gauge_flow_kernel(const __grid_constant__ GaugeFlowArgs<T> a)
  {
    const int x_cb = blockIdx.x * blockDim.x + threadIdx.x;
    if (x_cb >= a.f.g.volume_cb) return;
    gauge_flow_site(a, x_cb, blockIdx.z, blockIdx.y);
  }

  // partial[kind][parity][blockIdx.x] = the CTA's sums of E_spatial (kind 0), E_temporal (kind 1) and q (kind 2)
  template <typename T>
  __global__ void __launch_bounds__(kGaugeThreads) gauge_obs_kernel(const __grid_constant__ CloverBuildArgs<T> a, double *density, double *partial)
  {
    __shared__ double s[3][kGaugeThreads];
    const int tid = threadIdx.x, x_cb = blockIdx.x * blockDim.x + tid, parity = blockIdx.y;
    double sp = 0.0, tm = 0.0, q = 0.0;
    if (x_cb < a.volume_cb) {
      gauge_obs_site(a, x_cb, parity, sp, tm, q);
      if (density) density[(size_t)parity * a.volume_cb + x_cb] = q;
    }
    s[0][tid] = sp;
    s[1][tid] = tm;
    s[2][tid] = q;
    __syncthreads();
#pragma unroll
    for (int w = kGaugeThreads / 2; w > 0; w >>= 1) {
      clover_tree_step(s[0], tid, w);
      clover_tree_step(s[1], tid, w);
      clover_tree_step(s[2], tid, w);
      __syncthreads();
    }
    if (tid == 0) {
#pragma unroll
      for (int k = 0; k < 3; k++) partial[(k * 2 + parity) * gridDim.x + blockIdx.x] = s[k][0];
    }
  }

  template <typename T> int launch_gauge_flow(const GaugeFlowRequest &rq)
  {
    const size_t V = (size_t)rq.X[0] * rq.X[1] * rq.X[2] * rq.X[3];
    const int volume_cb = (int)(V / 2);
    const int nblk = (volume_cb + kGaugeThreads - 1) / kGaugeThreads;
    cudaStream_t st = (cudaStream_t)rq.stream;
    T *scratch = nullptr; // [4][V][18] links, then the accumulator [V][4][10]
    if (int rc = check_cuda(cudaMallocAsync((void **)&scratch, (4 * 18 + 4 * 10) * V * sizeof(T), st), "cudaMallocAsync")) return rc;
    void *tmp[4];
    for (int d = 0; d < 4; d++) tmp[d] = scratch + d * V * 18;
    void *acc = scratch + 4 * V * 18;
    const FlowPlan plan = flow_plan(rq);
    int rc = 0;
    const void *src[4];
    for (int d = 0; d < 4; d++) src[d] = rq.in[d];
    for (int s = 0; s < plan.stages && !rc; s++) {
      void *const *dst = plan.writes_scratch(s) ? tmp : rq.out;
      GaugeFlowArgs<T> a;
      fill_flow_stage(a, rq, s, src, dst, acc);
      gauge_flow_kernel<T><<<dim3(nblk, 4, 2), kGaugeThreads, 0, st>>>(a);
      count_launch();
      rc = check_cuda(cudaGetLastError(), "gauge flow launch");
      for (int d = 0; d < 4; d++) src[d] = dst[d];
    }
    if (!rc && plan.ends_in_scratch())
      for (int d = 0; d < 4 && !rc; d++)
        rc = check_cuda(cudaMemcpyAsync(rq.out[d], tmp[d], V * 18 * sizeof(T), cudaMemcpyDeviceToDevice, st), "flow copy");
    const int rf = check_cuda(cudaFreeAsync(scratch, st), "cudaFreeAsync");
    return rc ? rc : rf;
  }

  template <typename T> int launch_gauge_observables(const GaugeObsRequest &rq, double g[6])
  {
    CloverBuildArgs<T> a;
    fill_lattice(a, rq.qdp, rq.X);
    const int nblk = (a.volume_cb + kGaugeThreads - 1) / kGaugeThreads;
    cudaStream_t s = (cudaStream_t)rq.stream;
    double *scratch = nullptr; // [3][2][nblk] partials, then the six sums
    if (int rc = check_cuda(cudaMallocAsync((void **)&scratch, (6 * (size_t)nblk + 6) * sizeof(double), s), "cudaMallocAsync")) return rc;
    gauge_obs_kernel<T><<<dim3(nblk, 2, 1), kGaugeThreads, 0, s>>>(a, rq.density, scratch);
    count_launch();
    return finish_sums(scratch, nblk, 6, g, s);
  }

  template int launch_gauge_flow<double>(const GaugeFlowRequest &);
  template int launch_gauge_flow<float>(const GaugeFlowRequest &);
  template int launch_gauge_observables<double>(const GaugeObsRequest &, double *);
  template int launch_gauge_observables<float>(const GaugeObsRequest &, double *);

} // namespace b200
