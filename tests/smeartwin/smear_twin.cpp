// TEST-ONLY host twin of gauge smearing: twin_gauge_smear forwards to the same entry-point template as libquda_b200's
// b200_gauge_smear (quda_b200/csrc/gauge_smear.h: argument validation, site code, launch sequence) with a CPU executor that
// walks the grids of the kernels of inst_gauge_smear.cu site by site, level by level, on scratch poisoned with NaN.  It is
// built on the flow twin (tests/flowtwin), whose executor and entry points it includes, so one library also serves the
// gauge force, update, flow and observables the smearing tests call.  twin_su3_project exposes the projection alone.
// Nothing under quda_b200/ loads it.
#include "../../quda_b200/csrc/gauge_smear.h"
#include "../flowtwin/flow_twin.cpp"

namespace b200
{
  // the executor of run_gauge_smear: each launch is a grid (blocks, ndir, parity) in which every thread writes only its own
  // links
  struct SmearGrid {
    template <typename T> int stout(const GaugeStoutArgs<T> &a, int ndir)
    {
      for (int parity = 0; parity < 2; parity++)
        for (int yi = 0; yi < ndir; yi++)
#pragma omp parallel for
          for (int x_cb = 0; x_cb < a.f.g.volume_cb; x_cb++) gauge_stout_site(a, x_cb, parity, smear_dir(yi, a.ign));
      return 0;
    }
    template <typename T> int level(const SmearLevelArgs<T> &a, int ndir)
    {
      for (int parity = 0; parity < 2; parity++)
        for (int yi = 0; yi < ndir; yi++)
#pragma omp parallel for
          for (int x_cb = 0; x_cb < a.g.volume_cb; x_cb++) gauge_smear_level_site(a, x_cb, parity, smear_dir(yi, a.ign));
      return 0;
    }
    int copy(void *dst, const void *src, size_t bytes)
    {
      std::memmove(dst, src, bytes);
      return 0;
    }
  };

  struct SmearTwin : FlowTwin {
    template <typename T> static int gauge_smear(const GaugeSmearRequest &rq)
    {
      const size_t V = (size_t)rq.X[0] * rq.X[1] * rq.X[2] * rq.X[3];
      std::vector<T> scratch(smear_scratch_links(rq) * V * 18, std::numeric_limits<T>::quiet_NaN()); // as uninitialised memory
      SmearGrid x;
      return run_gauge_smear<T>(rq, scratch.data(), x);
    }
  };
} // namespace b200

extern "C" {
int twin_gauge_smear(void *const out[4], const void *const in[4], const int X[4], int precision, int type, const double coeff[3],
                     int dir_ignore, int n_steps, void *stream)
{
  return gauge_smear<SmearTwin>(out, in, X, precision, type, coeff, dir_ignore, n_steps, stream);
}

// p[n] = su3_project(w[n]) for n 3x3 complex matrices [n][3][3][2], in double (precision 8) or float (4), at the library's
// tolerance
int twin_su3_project(void *p, const void *w, int n, int precision)
{
  if (!p || !w || n < 0 || (precision != 8 && precision != 4)) return set_error(B200_ERR_INVALID, "twin_su3_project: bad argument");
  for (int i = 0; i < n; i++) {
    if (precision == 8) su3_project((double *)p + 18 * i, (const double *)w + 18 * i, kProjectTol<double>);
    else su3_project((float *)p + 18 * i, (const float *)w + 18 * i, kProjectTol<float>);
  }
  return 0;
}
}
