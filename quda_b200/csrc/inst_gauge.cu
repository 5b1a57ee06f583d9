// Kernels of b200_gauge_force, b200_update_gauge, b200_mom_action and b200_plaquette (site code: gauge.h).  The force and
// the update run one thread per (site, direction, parity) link; the two sums run one thread per site and reduce in two
// fixed-order stages (per-CTA trees here, then clover_trlog_kernel's strided sum and tree per group), so repeated calls give
// bit-identical results.
#include "gauge.h"

namespace b200
{

  // inst_clover_build.cu: out[g] = fixed-order sum of the n partials of group g = blockIdx.x (one CTA per group)
  __global__ void clover_trlog_kernel(const double *partial, int n, double *trlog);

  template <typename T> __global__ void __launch_bounds__(kGaugeThreads) gauge_force_kernel(const __grid_constant__ GaugeForceArgs<T> a)
  {
    const int x_cb = blockIdx.x * blockDim.x + threadIdx.x;
    if (x_cb >= a.g.volume_cb) return;
    gauge_force_site(a, x_cb, blockIdx.z, blockIdx.y);
  }

  template <typename T> __global__ void __launch_bounds__(kGaugeThreads) gauge_update_kernel(const __grid_constant__ GaugeUpdateArgs<T> a)
  {
    const int x_cb = blockIdx.x * blockDim.x + threadIdx.x;
    if (x_cb >= a.volume_cb) return;
    gauge_update_site(a, x_cb, blockIdx.z, blockIdx.y);
  }

  // partial[parity][blockIdx.x] = the CTA's sum of the momentum action
  template <typename T> __global__ void __launch_bounds__(kGaugeThreads) mom_action_kernel(const T *mom, int volume_cb, double *partial)
  {
    __shared__ double s[kGaugeThreads];
    const int tid = threadIdx.x, x_cb = blockIdx.x * blockDim.x + tid, parity = blockIdx.y;
    s[tid] = x_cb < volume_cb ? mom_action_site(mom, (size_t)parity * volume_cb + x_cb) : 0.0;
    __syncthreads();
#pragma unroll
    for (int w = kGaugeThreads / 2; w > 0; w >>= 1) {
      clover_tree_step(s, tid, w);
      __syncthreads();
    }
    if (tid == 0) partial[parity * gridDim.x + blockIdx.x] = s[0];
  }

  // partial[kind][parity][blockIdx.x] = the CTA's sums of Re tr over the spatial (kind 0) and temporal (kind 1) plaquettes
  template <typename T> __global__ void __launch_bounds__(kGaugeThreads) plaquette_kernel(const __grid_constant__ CloverBuildArgs<T> a, double *partial)
  {
    __shared__ double s[2][kGaugeThreads];
    const int tid = threadIdx.x, x_cb = blockIdx.x * blockDim.x + tid, parity = blockIdx.y;
    double sp = 0.0, tm = 0.0;
    if (x_cb < a.volume_cb) plaquette_site(a, x_cb, parity, sp, tm);
    s[0][tid] = sp;
    s[1][tid] = tm;
    __syncthreads();
#pragma unroll
    for (int w = kGaugeThreads / 2; w > 0; w >>= 1) {
      clover_tree_step(s[0], tid, w);
      clover_tree_step(s[1], tid, w);
      __syncthreads();
    }
    if (tid == 0) {
      partial[(0 * 2 + parity) * gridDim.x + blockIdx.x] = s[0][0];
      partial[(1 * 2 + parity) * gridDim.x + blockIdx.x] = s[1][0];
    }
  }

  template <typename T> int launch_gauge_force(const GaugeForceRequest &rq)
  {
    GaugeForceArgs<T> a;
    fill_gauge_force(a, rq);
    const int nblk = (a.g.volume_cb + kGaugeThreads - 1) / kGaugeThreads;
    gauge_force_kernel<T><<<dim3(nblk, 4, 2), kGaugeThreads, 0, (cudaStream_t)rq.stream>>>(a);
    count_launch();
    return check_cuda(cudaGetLastError(), "gauge force launch");
  }

  template <typename T> int launch_gauge_update(const GaugeUpdateRequest &rq)
  {
    GaugeUpdateArgs<T> a;
    fill_gauge_update(a, rq);
    const int nblk = (a.volume_cb + kGaugeThreads - 1) / kGaugeThreads;
    gauge_update_kernel<T><<<dim3(nblk, 4, 2), kGaugeThreads, 0, (cudaStream_t)rq.stream>>>(a);
    count_launch();
    return check_cuda(cudaGetLastError(), "gauge update launch");
  }

  // the second stage and the copy of the `groups` sums to the host, then the scratch is freed and the stream synchronised
  // (also the last step of inst_gauge_flow.cu's observables)
  int finish_sums(double *scratch, int nblk, int groups, double *g, cudaStream_t s)
  {
    clover_trlog_kernel<<<groups, kGaugeThreads, 0, s>>>(scratch, nblk, scratch + (size_t)groups * nblk);
    count_launch();
    int rc = check_cuda(cudaGetLastError(), "gauge sum launch");
    if (!rc) rc = check_cuda(cudaMemcpyAsync(g, scratch + (size_t)groups * nblk, groups * sizeof(double), cudaMemcpyDeviceToHost, s), "sum copy");
    const int rf = check_cuda(cudaFreeAsync(scratch, s), "cudaFreeAsync");
    if (!rc) rc = rf;
    if (!rc) rc = check_cuda(cudaStreamSynchronize(s), "gauge sum");
    return rc;
  }

  template <typename T> int launch_mom_action(const GaugeSumRequest &rq, double g[2])
  {
    const int volume_cb = rq.X[0] * rq.X[1] * rq.X[2] * rq.X[3] / 2;
    const int nblk = (volume_cb + kGaugeThreads - 1) / kGaugeThreads;
    cudaStream_t s = (cudaStream_t)rq.stream;
    double *scratch = nullptr; // [2][nblk] partials, then the two sums
    if (int rc = check_cuda(cudaMallocAsync((void **)&scratch, (2 * (size_t)nblk + 2) * sizeof(double), s), "cudaMallocAsync")) return rc;
    mom_action_kernel<T><<<dim3(nblk, 2, 1), kGaugeThreads, 0, s>>>((const T *)rq.mom, volume_cb, scratch);
    count_launch();
    return finish_sums(scratch, nblk, 2, g, s);
  }

  template <typename T> int launch_plaquette(const GaugeSumRequest &rq, double g[4])
  {
    CloverBuildArgs<T> a;
    fill_lattice(a, rq.qdp, rq.X);
    const int nblk = (a.volume_cb + kGaugeThreads - 1) / kGaugeThreads;
    cudaStream_t s = (cudaStream_t)rq.stream;
    double *scratch = nullptr; // [2][2][nblk] partials, then the four sums
    if (int rc = check_cuda(cudaMallocAsync((void **)&scratch, (4 * (size_t)nblk + 4) * sizeof(double), s), "cudaMallocAsync")) return rc;
    plaquette_kernel<T><<<dim3(nblk, 2, 1), kGaugeThreads, 0, s>>>(a, scratch);
    count_launch();
    return finish_sums(scratch, nblk, 4, g, s);
  }

  template int launch_gauge_force<double>(const GaugeForceRequest &);
  template int launch_gauge_force<float>(const GaugeForceRequest &);
  template int launch_gauge_update<double>(const GaugeUpdateRequest &);
  template int launch_gauge_update<float>(const GaugeUpdateRequest &);
  template int launch_mom_action<double>(const GaugeSumRequest &, double *);
  template int launch_mom_action<float>(const GaugeSumRequest &, double *);
  template int launch_plaquette<double>(const GaugeSumRequest &, double *);
  template int launch_plaquette<float>(const GaugeSumRequest &, double *);

} // namespace b200
