// Kernels of b200_gauge_smear (site code and launch sequence: gauge_smear.h).  One thread per (site, smeared direction,
// parity) link, CTAs of kGaugeThreads, grid (blocks, smeared directions, parity); one launch per step, and for HYP one per
// level and step.  Decorated HYP links and the ping-pong link field live in one stream-ordered scratch allocation.
#include "gauge_smear.h"

namespace b200
{

  template <typename T> __global__ void __launch_bounds__(kGaugeThreads) gauge_stout_kernel(const __grid_constant__ GaugeStoutArgs<T> a)
  {
    const int x_cb = blockIdx.x * blockDim.x + threadIdx.x;
    if (x_cb >= a.f.g.volume_cb) return;
    gauge_stout_site(a, x_cb, blockIdx.z, smear_dir(blockIdx.y, a.ign));
  }

  template <typename T>
  __global__ void __launch_bounds__(kGaugeThreads) gauge_smear_level_kernel(const __grid_constant__ SmearLevelArgs<T> a)
  {
    const int x_cb = blockIdx.x * blockDim.x + threadIdx.x;
    if (x_cb >= a.g.volume_cb) return;
    gauge_smear_level_site(a, x_cb, blockIdx.z, smear_dir(blockIdx.y, a.ign));
  }

  struct CudaSmear {
    cudaStream_t st;
    int nblk;
    template <typename T> int stout(const GaugeStoutArgs<T> &a, int ndir)
    {
      gauge_stout_kernel<T><<<dim3(nblk, ndir, 2), kGaugeThreads, 0, st>>>(a);
      count_launch();
      return check_cuda(cudaGetLastError(), "gauge stout launch");
    }
    template <typename T> int level(const SmearLevelArgs<T> &a, int ndir)
    {
      gauge_smear_level_kernel<T><<<dim3(nblk, ndir, 2), kGaugeThreads, 0, st>>>(a);
      count_launch();
      return check_cuda(cudaGetLastError(), "gauge smear launch");
    }
    int copy(void *dst, const void *src, size_t bytes)
    {
      return check_cuda(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st), "smear copy");
    }
  };

  template <typename T> int launch_gauge_smear(const GaugeSmearRequest &rq)
  {
    const size_t V = (size_t)rq.X[0] * rq.X[1] * rq.X[2] * rq.X[3];
    CudaSmear x {(cudaStream_t)rq.stream, (int)((V / 2 + kGaugeThreads - 1) / kGaugeThreads)};
    const size_t bytes = smear_scratch_links(rq) * V * 18 * sizeof(T); // 0: one APE or stout step out of place
    T *scratch = nullptr;
    if (bytes)
      if (int rc = check_cuda(cudaMallocAsync((void **)&scratch, bytes, x.st), "cudaMallocAsync")) return rc;
    const int rc = run_gauge_smear<T>(rq, scratch, x);
    const int rf = bytes ? check_cuda(cudaFreeAsync(scratch, x.st), "cudaFreeAsync") : 0;
    return rc ? rc : rf;
  }

  template int launch_gauge_smear<double>(const GaugeSmearRequest &);
  template int launch_gauge_smear<float>(const GaugeSmearRequest &);

} // namespace b200
