// Kernels of b200_compute_clover and b200_clover_invert_packed (site code: clover_build.h).  One thread per site; the
// trlog reduction is two-stage in a fixed order (per-CTA trees, then one CTA per parity over the CTA partials), so
// repeated calls give bit-identical sums.
#include "clover_build.h"

namespace b200
{

  template <typename T> __global__ void __launch_bounds__(kCloverBuildThreads) clover_build_kernel(const CloverBuildArgs<T> a)
  {
    const int x_cb = blockIdx.x * blockDim.x + threadIdx.x;
    if (x_cb >= a.volume_cb) return;
    clover_build_site(a, x_cb, blockIdx.y);
  }

  // partial[parity][blockIdx.x] = sum of log det A over the CTA's sites
  template <typename T>
  __global__ void __launch_bounds__(kCloverBuildThreads) clover_invert_kernel(T *inv, const T *packed, int volume_cb, double *partial)
  {
    __shared__ double s[kCloverBuildThreads];
    const int tid = threadIdx.x, x_cb = blockIdx.x * blockDim.x + tid, parity = blockIdx.y;
    s[tid] = x_cb < volume_cb ? clover_invert_site(inv, packed, (size_t)parity * volume_cb + x_cb) : 0.0;
    __syncthreads();
#pragma unroll
    for (int w = kCloverBuildThreads / 2; w > 0; w >>= 1) {
      clover_tree_step(s, tid, w);
      __syncthreads();
    }
    if (tid == 0) partial[parity * gridDim.x + blockIdx.x] = s[0];
  }

  // trlog[parity] = sum of the n CTA partials of that parity (one CTA per parity)
  __global__ void __launch_bounds__(kCloverBuildThreads) clover_trlog_kernel(const double *partial, int n, double *trlog)
  {
    __shared__ double s[kCloverBuildThreads];
    const int tid = threadIdx.x, parity = blockIdx.x;
    double v = 0.0;
    for (int i = tid; i < n; i += kCloverBuildThreads) v += partial[parity * n + i];
    s[tid] = v;
    __syncthreads();
#pragma unroll
    for (int w = kCloverBuildThreads / 2; w > 0; w >>= 1) {
      clover_tree_step(s, tid, w);
      __syncthreads();
    }
    if (tid == 0) trlog[parity] = s[0];
  }

  template <typename T> int launch_clover_build(const CloverBuildRequest &rq)
  {
    CloverBuildArgs<T> a;
    fill_clover_build(a, rq);
    const dim3 grid((a.volume_cb + kCloverBuildThreads - 1) / kCloverBuildThreads, 2, 1);
    clover_build_kernel<T><<<grid, kCloverBuildThreads, 0, (cudaStream_t)rq.stream>>>(a);
    count_launch();
    return check_cuda(cudaGetLastError(), "clover build launch");
  }

  template <typename T> int launch_clover_invert(const CloverInvertRequest &rq)
  {
    const int volume_cb = rq.X[0] * rq.X[1] * rq.X[2] * rq.X[3] / 2;
    const int nblk = (volume_cb + kCloverBuildThreads - 1) / kCloverBuildThreads;
    cudaStream_t s = (cudaStream_t)rq.stream;
    double *scratch = nullptr; // [2][nblk] partials, then the two sums
    if (int rc = check_cuda(cudaMallocAsync((void **)&scratch, (2 * (size_t)nblk + 2) * sizeof(double), s), "cudaMallocAsync")) return rc;
    clover_invert_kernel<T><<<dim3(nblk, 2, 1), kCloverBuildThreads, 0, s>>>((T *)rq.inv, (const T *)rq.packed, volume_cb, scratch);
    count_launch();
    clover_trlog_kernel<<<2, kCloverBuildThreads, 0, s>>>(scratch, nblk, scratch + 2 * nblk);
    count_launch();
    int rc = check_cuda(cudaGetLastError(), "clover invert launch");
    if (!rc) rc = check_cuda(cudaMemcpyAsync(rq.trlog, scratch + 2 * nblk, 2 * sizeof(double), cudaMemcpyDeviceToHost, s), "trlog copy");
    const int rf = check_cuda(cudaFreeAsync(scratch, s), "cudaFreeAsync");
    if (!rc) rc = rf;
    if (!rc) rc = check_cuda(cudaStreamSynchronize(s), "clover invert");
    return rc;
  }

  template int launch_clover_build<double>(const CloverBuildRequest &);
  template int launch_clover_build<float>(const CloverBuildRequest &);
  template int launch_clover_invert<double>(const CloverInvertRequest &);
  template int launch_clover_invert<float>(const CloverInvertRequest &);

} // namespace b200
