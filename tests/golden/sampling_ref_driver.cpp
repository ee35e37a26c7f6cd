// extern "C" entry points that run the reference's own joint posterior sampling on a GaussianProcess made by
// oracle/_ref/libmoe_ref.so (ref_gp_create).  Used only by make_sampling_golden.py, which compiles this file against
// the reference headers and links it to oracle/_ref/libmoe_ref.so; the product never sees it.
//
// Both calls reseed first: GaussianProcess::SetExplicitSeed -> NormalRNG::SetExplicitSeed, which also resets the
// distribution (gpp_random.cpp:91-121), so the normals consumed are the first Q draws of NormalRNG(seed) — the table
// ref_normal_draws(seed, Q) returns.
#include "gpp_math.hpp"

using optimal_learning::GaussianProcess;

extern "C" {

// GaussianProcess::SamplePointsFromGP (gpp_math.cpp:1803-1848): results[num]; returns the reference's best_point
// (-1 when point 0 is the minimum).
int sref_sample_points(void* h, unsigned seed, const double* points, int num, double* results) {
  auto* gp = static_cast<GaussianProcess*>(h);
  gp->SetExplicitSeed(seed);
  return gp->SamplePointsFromGP(points, num, results);
}

// GaussianProcess::SamplePointFromGP (gpp_math.cpp:1761-1798): results[1 + num_derivatives] at one point.
void sref_sample_point(void* h, unsigned seed, const double* point, double* results) {
  auto* gp = static_cast<GaussianProcess*>(h);
  gp->SetExplicitSeed(seed);
  gp->SamplePointFromGP(point, results);
}

}  // extern "C"
