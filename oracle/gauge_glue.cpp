/*
 * TEST INFRASTRUCTURE ONLY -- exports of oracle/_ref/libquda_gaugeref.so (gauge_ref.mk).
 *
 * Forwards to the reference's own host code, compiled in place:
 *   tests/host_reference/gauge_force_reference.cpp  gauge_force_reference_dir (the momentum update from a path table)
 *   tests/utils/host_utils.cpp                      mom_action (MILC's momentum action)
 * ref_glue.cpp supplies the link-time stand-ins.  No reference source text is copied.
 */
#include <cstddef>
#include <vector>

#include <quda.h>
#include <host_utils.h>
#include <gauge_force_reference.h>

#define EXPORT extern "C" __attribute__((visibility("default")))

// defined (not declared in the header) in tests/host_reference/gauge_force_reference.cpp
void gauge_force_reference_dir(void *refMom, int dir, double eb3, void *const *sitelink, void *const *sitelink_ex,
                               QudaPrecision prec, int **path_dir, int *length, void *loop_coeff, int num_paths,
                               const lattice_t &lat, bool compute_force);

namespace
{
  /* lattice_t can only be constructed from a quda::GaugeField; this struct has its layout (unextended lattice: r = 0,
     e = x) and is handed over in its place */
  struct lattice_layout {
    int n_color;
    size_t volume;
    size_t volume_ex;
    int x[4];
    int r[4];
    int e[4];
  };
  static_assert(sizeof(lattice_layout) == sizeof(lattice_t), "lattice_t layout");
  static_assert(offsetof(lattice_layout, e) == offsetof(lattice_t, e), "lattice_t layout");
} // namespace

/* mom [V][4][10] += the reference's gauge force, fp64, one unpartitioned lattice X; paths flat [4][num_paths][max_length].
   ref_set_dims(X) must have been called: the reference sizes its staple buffer from the global V. */
EXPORT void ref_gauge_force(double *mom, void **gauge, const int *X, const int *paths, const int *length, const double *coeff,
                            int num_paths, int max_length, double eb3)
{
  lattice_layout lat;
  lat.n_color = 3;
  lat.volume = 1;
  for (int d = 0; d < 4; d++) {
    lat.x[d] = X[d];
    lat.r[d] = 0;
    lat.e[d] = X[d];
    lat.volume *= X[d];
  }
  lat.volume_ex = lat.volume;
  std::vector<int> table(paths, paths + (size_t)4 * num_paths * max_length), len(length, length + num_paths);
  std::vector<double> c(coeff, coeff + num_paths);
  std::vector<int *> rows(num_paths);
  for (int dir = 0; dir < 4; dir++) {
    for (int i = 0; i < num_paths; i++) rows[i] = table.data() + ((size_t)dir * num_paths + i) * max_length;
    gauge_force_reference_dir(mom, dir, eb3, gauge, gauge, QUDA_DOUBLE_PRECISION, rows.data(), len.data(), c.data(), num_paths,
                              *reinterpret_cast<const lattice_t *>(&lat), true);
  }
}

/* sum over the n links of mom[n][10] of the MILC momentum action, in the precision of mom (8 or 4 bytes) */
EXPORT double ref_mom_action(void *mom, int prec_bytes, int n_links)
{
  return mom_action(mom, prec_bytes == 8 ? QUDA_DOUBLE_PRECISION : QUDA_SINGLE_PRECISION, n_links);
}
