// TEST-ONLY host twin of the gauge half of an HMC step: twin_gauge_force / twin_update_gauge / twin_mom_action /
// twin_plaquette forward to the same entry-point templates as libquda_b200's b200_gauge_force / b200_update_gauge /
// b200_mom_action / b200_plaquette (quda_b200/csrc/gauge.h: argument validation, site code) with a CPU executor that walks
// the grids of the kernels of inst_gauge.cu site by site, and sums in the kernels' order.  It exists so that the CPU test
// tier checks the code the GPU runs; nothing under quda_b200/ loads it.
#include <cstdarg>
#include <cstdio>
#include <vector>

#include "../../quda_b200/csrc/gauge.h"

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

  struct GaugeTwin {
    static int require_device() { return 0; }

    // gauge_force_kernel: grid (blocks, mu, parity)
    template <typename T> static int gauge_force(const GaugeForceRequest &rq)
    {
      GaugeForceArgs<T> a;
      fill_gauge_force(a, rq);
      for (int parity = 0; parity < 2; parity++)
        for (int mu = 0; mu < 4; mu++)
#pragma omp parallel for
          for (int x_cb = 0; x_cb < a.g.volume_cb; x_cb++) gauge_force_site(a, x_cb, parity, mu);
      return 0;
    }

    // gauge_update_kernel: grid (blocks, mu, parity); every thread reads and writes only its own link
    template <typename T> static int gauge_update(const GaugeUpdateRequest &rq)
    {
      GaugeUpdateArgs<T> a;
      fill_gauge_update(a, rq);
      for (int parity = 0; parity < 2; parity++)
        for (int mu = 0; mu < 4; mu++)
#pragma omp parallel for
          for (int x_cb = 0; x_cb < a.volume_cb; x_cb++) gauge_update_site(a, x_cb, parity, mu);
      return 0;
    }

    // The two reduction stages of inst_gauge.cu: per-CTA trees over kGaugeThreads sites (site(x_cb, parity, kind) for
    // `kinds` values per site), then one CTA per (kind, parity) group that strides over the CTA partials and reduces them
    // with the same tree (clover_trlog_kernel)
    template <class Site> static void two_stage(int volume_cb, int kinds, double *g, Site site)
    {
      constexpr int B = kGaugeThreads;
      const int nblk = (volume_cb + B - 1) / B;
      std::vector<double> partial((size_t)kinds * 2 * nblk);
      auto tree = [](double *s) {
        for (int w = B / 2; w > 0; w >>= 1)
          for (int tid = 0; tid < B; tid++) clover_tree_step(s, tid, w);
      };
      for (int parity = 0; parity < 2; parity++)
#pragma omp parallel for
        for (int b = 0; b < nblk; b++) {
          double s[2][B];
          for (int tid = 0; tid < B; tid++) {
            const int x_cb = b * B + tid;
            double v[2] = {0.0, 0.0};
            if (x_cb < volume_cb) site(x_cb, parity, v);
            for (int k = 0; k < kinds; k++) s[k][tid] = v[k];
          }
          for (int k = 0; k < kinds; k++) {
            tree(s[k]);
            partial[((size_t)k * 2 + parity) * nblk + b] = s[k][0];
          }
        }
      for (int grp = 0; grp < 2 * kinds; grp++) {
        double s[B];
        for (int tid = 0; tid < B; tid++) {
          double v = 0.0;
          for (int i = tid; i < nblk; i += B) v += partial[(size_t)grp * nblk + i];
          s[tid] = v;
        }
        tree(s);
        g[grp] = s[0];
      }
    }

    template <typename T> static int mom_action(const GaugeSumRequest &rq, double g[2])
    {
      const int volume_cb = rq.X[0] * rq.X[1] * rq.X[2] * rq.X[3] / 2;
      const T *mom = reinterpret_cast<const T *>(rq.mom);
      two_stage(volume_cb, 1, g, [&](int x_cb, int parity, double *v) { v[0] = mom_action_site(mom, (size_t)parity * volume_cb + x_cb); });
      return 0;
    }

    template <typename T> static int plaquette(const GaugeSumRequest &rq, double g[4])
    {
      CloverBuildArgs<T> a;
      fill_lattice(a, rq.qdp, rq.X);
      two_stage(a.volume_cb, 2, g, [&](int x_cb, int parity, double *v) { plaquette_site(a, x_cb, parity, v[0], v[1]); });
      return 0;
    }
  };
} // namespace b200

using namespace b200;

extern "C" {
const char *twin_last_error(void) { return g_err; }

int twin_gauge_force(void *mom, const void *const qdp[4], const int X[4], int precision, const int *paths, const int *length,
                     const double *coeff, int num_paths, int max_length, double eb3, void *stream)
{
  return gauge_force<GaugeTwin>(mom, qdp, X, precision, paths, length, coeff, num_paths, max_length, eb3, stream);
}

int twin_update_gauge(void *const out[4], const void *const in[4], const void *mom, const int X[4], int precision, double dt,
                      int conj_mom, int exact, void *stream)
{
  return update_gauge<GaugeTwin>(out, in, mom, X, precision, dt, conj_mom, exact, stream);
}

int twin_mom_action(double *S, const void *mom, const int X[4], int precision, void *stream)
{
  return mom_action<GaugeTwin>(S, mom, X, precision, stream);
}

int twin_plaquette(double plaq[3], const void *const qdp[4], const int X[4], int precision, void *stream)
{
  return plaquette<GaugeTwin>(plaq, qdp, X, precision, stream);
}
}
