// Multistart optimisation drivers: screen every start, keep the best 20, run restarted gradient descent on those
// (all starts advance together, one batched device evaluation per step), strict-> arg-max.
//
// Replaces (reference, moe/optimal_learning/cpp/):
//   ComputeKGOptimalPointsToSampleViaMultistartGradientDescent   gpp_knowledge_gradient_optimization.hpp:859-935
//   ComputeOptimalPointsToSampleViaMultistartGradientDescent     gpp_math.hpp:1683-1802
//   GradientDescentOptimization / GradientDescentOptimizer::Optimize   gpp_optimization.hpp:620-705, 1144-1185
//   MultistartOptimizer::MultistartOptimize (arg-max part)        gpp_optimization.hpp:1452-1564
//   RepeatedDomain::LimitUpdate / TensorProductDomain::LimitUpdate gpp_domain.hpp:536-540, gpp_domain.cpp:64-104
//   OnePotentialSampleExpectedImprovementEvaluator                gpp_math.cpp:2196-2253
// The step bookkeeping is O(q*dim) per start and stays on the host; every objective / gradient evaluation is a
// batched device call (kg.cu / ei.cu / posterior.cu).
#include <algorithm>
#include <cmath>
#include <functional>
#include <limits>
#include <memory>
#include <exception>
#include <queue>
#include <thread>

#include "device_math.cuh"
#include "internal.cuh"

using namespace cmoe;  // NOLINT

namespace {

// SimplexIntersectTensorProductDomain::LimitUpdate (gpp_domain.cpp:234-289) for one point: box limited to [0,1]^dim
// (constructor, :107-139), tensor-product limit first, then half the distance to the diagonal face if the limited step
// would leave the simplex.
void limit_update_simplex_host(const double* bounds, int dim, double mrc, const double* x, double* upd) {
  if (mrc == 1.0) mrc -= 4.0 * std::numeric_limits<double>::epsilon();  // kRelativeChangeEpsilonTweak
  for (int d = 0; d < dim; ++d) {
    const double lo = std::fmax(bounds[2 * d], 0.0), hi = std::fmin(bounds[2 * d + 1], 1.0);
    upd[d] = limit_step(upd[d], x[d], lo, hi, mrc);
  }
  double norm = 0.0;
  for (int d = 0; d < dim; ++d) norm += upd[d] * upd[d];
  norm = std::sqrt(norm);
  if (norm == 0.0) norm = std::numeric_limits<double>::min();
  bool inside = true;
  double sum = 0.0;
  for (int d = 0; d < dim; ++d) {
    const double t = x[d] + upd[d];
    if (t < 0.0) inside = false;
    sum += t;
  }
  inside = inside && (sum - 4.0 * std::numeric_limits<double>::epsilon()) <= 1.0;  // CheckPointInUnitSimplex
  if (!inside) {
    // plane -1/sqrt(dim) + sum_i x_i / sqrt(dim) = 0; distance along the unit direction (gpp_geometry.hpp:252-272)
    const double nrm = 1.0 / std::sqrt(static_cast<double>(dim));
    double xn = 0.0, vn = 0.0;
    for (int d = 0; d < dim; ++d) {
      xn += x[d] * nrm;
      vn += (upd[d] / norm) * nrm;
    }
    const double numerator = nrm - xn;
    double dist = (vn == 0.0) ? ((numerator == 0.0) ? 0.0 : std::numeric_limits<double>::infinity()) : numerator / vn;
    if (dist < 0.0) dist = 0.0;
    const double step = 0.5 * dist;  // kInvalidStepScaleFactor
    for (int d = 0; d < dim; ++d) upd[d] = step * (upd[d] / norm);
  }
}

using BatchEval = std::function<void(const double* pts, int nc, double* values, double* grads)>;

// Restarted gradient descent on `ns` starts at once.  eval(pts, nc, values, grads): grads may be NULL.
void gradient_descent_batch(const BatchEval& eval, const cmoe_gd_params& gd, const double* domain_bounds, int q,
                            int dim, const double* starts, int ns, double* values_out, double* points_out,
                            int domain_type = CMOE_DOMAIN_TENSOR_PRODUCT) {
  const int ps = q * dim;
  std::vector<double> x(starts, starts + static_cast<size_t>(ns) * ps);
  if (gd.max_num_restarts > 0) {
    std::vector<char> converged(ns, 0);
    std::vector<double> x0(x.size()), pts, vals, grads;
    const double step_tol = gd.tolerance / static_cast<double>(gd.max_num_steps);
    for (int r = 0; r < gd.max_num_restarts; ++r) {
      std::vector<int> act;
      for (int s = 0; s < ns; ++s)
        if (!converged[s]) act.push_back(s);
      if (act.empty()) break;
      x0 = x;
      std::vector<char> run_done(ns, 0);
      for (int i = 0; i < gd.max_num_steps; ++i) {
        std::vector<int> cur;
        for (int s : act)
          if (!run_done[s]) cur.push_back(s);
        if (cur.empty()) break;
        const int nc = static_cast<int>(cur.size());
        pts.resize(static_cast<size_t>(nc) * ps);
        vals.resize(nc);
        grads.resize(static_cast<size_t>(nc) * ps);
        for (int k = 0; k < nc; ++k)
          std::copy(x.begin() + static_cast<size_t>(cur[k]) * ps, x.begin() + static_cast<size_t>(cur[k] + 1) * ps,
                    pts.begin() + static_cast<size_t>(k) * ps);
        eval(pts.data(), nc, vals.data(), grads.data());
        const double alpha = gd_step_size(gd.pre_mult, gd.gamma, i);
        for (int k = 0; k < nc; ++k) {
          double* xs = x.data() + static_cast<size_t>(cur[k]) * ps;
          const double* g = grads.data() + static_cast<size_t>(k) * ps;
          double ns2 = 0.0;
          if (domain_type == CMOE_DOMAIN_SIMPLEX) {
            // RepeatedDomain::LimitUpdate: each of the q points against the simplex domain (gpp_domain.hpp:536-540)
            double upd[CMOE_MAX_DIM];
            for (int pt = 0; pt < q; ++pt) {
              for (int d = 0; d < dim; ++d) upd[d] = alpha * g[pt * dim + d];
              limit_update_simplex_host(domain_bounds, dim, gd.max_relative_change, xs + pt * dim, upd);
              for (int d = 0; d < dim; ++d) {
                xs[pt * dim + d] += upd[d];
                ns2 += upd[d] * upd[d];
              }
            }
          } else {
            for (int j = 0; j < ps; ++j) {
              const int d = j % dim;
              const double step = limit_step(alpha * g[j], xs[j], domain_bounds[2 * d], domain_bounds[2 * d + 1],
                                                  gd.max_relative_change);
              xs[j] += step;
              ns2 += step * step;
            }
          }
          if (std::sqrt(ns2) < step_tol) run_done[cur[k]] = 1;
        }
      }
      for (int s : act) {
        double nd = 0.0;
        for (int j = 0; j < ps; ++j) {
          const double df = x0[static_cast<size_t>(s) * ps + j] - x[static_cast<size_t>(s) * ps + j];
          nd += df * df;
        }
        if (std::sqrt(nd) <= gd.tolerance) converged[s] = 1;
      }
    }
  }
  eval(x.data(), ns, values_out, nullptr);
  std::copy(x.begin(), x.end(), points_out);
}

}  // namespace

std::vector<int> cmoe::top_k_indices(const double* values, int n) {
  std::priority_queue<std::pair<double, int>> pq;
  const int k = std::min(kTopK, n);
  for (int i = 0; i < n; ++i) {
    if (i < k) {
      pq.push({-values[i], i});
    } else if (pq.top().first > -values[i]) {
      pq.pop();
      pq.push({-values[i], i});
    }
  }
  std::vector<int> out;
  while (!pq.empty()) {
    out.push_back(pq.top().second);
    pq.pop();
  }
  return out;
}

namespace {

void multistart_common(const BatchEval& eval, const cmoe_gd_params& outer, const double* domain_bounds, int q, int dim,
                       const double* starts, int num_starts, double init_best, double* start_values,
                       double* best_point, double* best_value, int* found_flag,
                       int domain_type = CMOE_DOMAIN_TENSOR_PRODUCT) {
  const int ps = q * dim;
  std::vector<double> vals(num_starts);
  eval(starts, num_starts, vals.data(), nullptr);
  if (start_values) std::copy(vals.begin(), vals.end(), start_values);
  const std::vector<int> top = top_k_indices(vals.data(), num_starts);
  const int k = static_cast<int>(top.size());
  std::vector<double> tk(static_cast<size_t>(k) * ps), fin_v(k), fin_p(static_cast<size_t>(k) * ps);
  for (int i = 0; i < k; ++i)
    std::copy(starts + static_cast<size_t>(top[i]) * ps, starts + static_cast<size_t>(top[i] + 1) * ps,
              tk.begin() + static_cast<size_t>(i) * ps);
  gradient_descent_batch(eval, outer, domain_bounds, q, dim, tk.data(), k, fin_v.data(), fin_p.data(), domain_type);
  // OptimizationIOContainer: best point initialised to the first start, strict `<` update
  double best = init_best;
  int found = 0;
  std::copy(tk.begin(), tk.begin() + ps, best_point);
  for (int i = 0; i < k; ++i) {
    if (best < fin_v[i]) {
      best = fin_v[i];
      found = 1;
      std::copy(fin_p.begin() + static_cast<size_t>(i) * ps, fin_p.begin() + static_cast<size_t>(i + 1) * ps,
                best_point);
    }
  }
  if (best_value) *best_value = best;
  if (found_flag) *found_flag = found;
}

// The q-KG evaluation of the drivers for an ensemble of num_gp >= 1 GPs (a single GP is the one-member ensemble): the
// members' values and gradients summed in member order.  Up to CMOE_MAX_KG_ROWS union rows, (q + p)(1 + g), each member
// has two plans (values, gradients); every member's plan is enqueued on its own stream before the first is drained.
// Past them one kg_large_eval call runs every member on the large-union stages, with the evaluation's arguments kept
// here.  Both paths use the same normals table and stale union.
struct KgEvaluator {
  std::vector<std::pair<cmoe_kg_plan*, cmoe_kg_plan*>> plans;  // (values, gradients) per member
  size_t ps = 0;
  std::vector<double> tv, tg;
  // large path: the evaluation's arguments (host copies)
  bool large = false;
  std::vector<const cmoe_gp*> gps;
  int nf = 0, num_pts = 0, q = 0, p = 0, num_mc = 0;
  uint64_t seed = 0;
  cmoe_gd_params inner{};
  std::vector<double> inner_bounds, discrete, Xp, best, stale, table;
  ~KgEvaluator() {
    for (auto& pp : plans) {
      cmoe_kg_plan_destroy(pp.first);
      cmoe_kg_plan_destroy(pp.second);
    }
  }
  static void check(int rc, int info = 0) {
    if (rc != CMOE_OK) throw Error(rc, cmoe_last_error(), info);
  }
  // replays `t` (NormalRNGSimulator semantics) in every evaluation
  void set_table(const double* t, size_t len) {
    if (!large) {
      for (auto& pp : plans) {
        check(cmoe_kg_plan_set_table(pp.first, t, static_cast<int>(len)));
        check(cmoe_kg_plan_set_table(pp.second, t, static_cast<int>(len)));
      }
      return;
    }
    const size_t need = static_cast<size_t>((num_mc + 1) / 2) * (q + p) * (1 + gps[0]->spec.g);
    CMOE_REQUIRE(len >= need, CMOE_ERR_INVALID_VALUE, "All random numbers stored in the RNG have been used up!");
    table.assign(t, t + need);
  }
  void operator()(const double* pts, int nc, double* values, double* grads) {
    if (large) {
      require_device(gps[0]->device);  // may run on a worker thread of the multi-device driver
      kg_large_eval(gps.data(), static_cast<int>(gps.size()), nf, &inner, inner_bounds.data(), discrete.data(),
                    num_pts, pts, nc, q, Xp.data(), p, num_mc, best.data(), seed,
                    table.empty() ? nullptr : table.data(), stale.empty() ? nullptr : stale.data(), values, grads,
                    nullptr);
      return;
    }
    for (auto& pp : plans) {
      cmoe_kg_plan* pl = grads ? pp.second : pp.first;
      check(cmoe_kg_plan_upload(pl, pts, nc));
      check(cmoe_kg_plan_run(pl));
    }
    tv.resize(nc);
    if (grads) tg.resize(nc * ps);
    for (size_t m = 0; m < plans.size(); ++m) {
      cmoe_kg_plan* pl = grads ? plans[m].second : plans[m].first;
      int info = 0;
      check(cmoe_kg_plan_sync(pl, &info), info);
      check(cmoe_kg_plan_download(pl, tv.data(), grads ? tg.data() : nullptr, nullptr));
      add_member(static_cast<int>(m), nc, ps, tv.data(), grads ? tg.data() : nullptr, values, grads);
    }
  }
};

void make_kg_evaluator(KgEvaluator& ev, const cmoe_gp* const* gps, int num_gp, int nf, const cmoe_gd_params* inner,
                       const double* inner_bounds, const double* discrete_pts, int num_pts, int max_value_cands,
                       int max_grad_cands, int q, const double* Xp, int p, int num_mc, const double* best_so_far,
                       uint64_t seed, const double* stale_union = nullptr) {
  const int dim = gps[0]->spec.dim, ps = dim - nf;
  ev.ps = static_cast<size_t>(q) * dim;
  if (kg_union_is_large(q, p, gps[0]->spec.g)) {
    CMOE_REQUIRE(nf >= 0 && ps >= 1 && num_pts >= 0, CMOE_ERR_BOUNDS, "num_fidelity out of range");
    ev.large = true;
    ev.gps.assign(gps, gps + num_gp);
    ev.nf = nf;
    ev.num_pts = num_pts;
    ev.q = q;
    ev.p = p;
    ev.num_mc = num_mc;
    ev.seed = seed;
    ev.inner = *inner;
    ev.inner_bounds.assign(inner_bounds, inner_bounds + 2 * static_cast<size_t>(ps));
    ev.discrete.assign(discrete_pts, discrete_pts + static_cast<size_t>(num_gp) * num_pts * ps);
    if (p) ev.Xp.assign(Xp, Xp + static_cast<size_t>(p) * dim);
    ev.best.assign(best_so_far, best_so_far + num_gp);
    if (stale_union) ev.stale.assign(stale_union, stale_union + static_cast<size_t>(q) * dim);
    return;
  }
  for (int m = 0; m < num_gp; ++m) {
    ev.plans.emplace_back(nullptr, nullptr);
    auto& pp = ev.plans.back();
    const double* disc = discrete_pts + static_cast<size_t>(m) * num_pts * ps;
    KgEvaluator::check(cmoe_kg_plan_create(gps[m], nf, inner, inner_bounds, disc, num_pts, max_value_cands, q, Xp, p,
                                           num_mc, best_so_far[m], seed, 0, &pp.first));
    KgEvaluator::check(cmoe_kg_plan_create(gps[m], nf, inner, inner_bounds, disc, num_pts, max_grad_cands, q, Xp, p,
                                           num_mc, best_so_far[m], seed, 1, &pp.second));
    if (stale_union) {
      KgEvaluator::check(cmoe_kg_plan_set_stale_union(pp.first, stale_union));
      KgEvaluator::check(cmoe_kg_plan_set_stale_union(pp.second, stale_union));
    }
  }
}

}  // namespace

void cmoe::analytic_ei(const cmoe_gp* gp, const double* pts, int nc, double best_so_far, double* values, double* grads) {
  const int dim = gp->spec.dim;
  std::vector<double> mu(nc), var(nc), gmu, gvar;
  int info = 0;
  if (grads) {
    gmu.resize(static_cast<size_t>(nc) * dim);
    gvar.resize(static_cast<size_t>(nc) * dim);
  }
  const int rc = cmoe_gp_posterior(gp, pts, nc, 1, nullptr, 0, mu.data(), grads ? gmu.data() : nullptr, var.data(),
                                   nullptr, grads ? gvar.data() : nullptr, nullptr, &info);
  if (rc != CMOE_OK) throw Error(rc, cmoe_last_error(), info);
  const double kMinVarEI = std::numeric_limits<double>::min();
  const double eps = std::numeric_limits<double>::epsilon();
  const double kMinVarGradEI = 150.0 * eps * eps;
  const double inv_sqrt_2pi = 0.39894228040143267793994605993438;
  auto pdf = [&](double z) { return std::exp(-0.5 * z * z) * inv_sqrt_2pi; };
  auto cdf = [&](double z) { return 0.5 * std::erfc(-z * 0.70710678118654752440084436210485); };
  for (int c = 0; c < nc; ++c) {
    {
      const double sigma = std::sqrt(std::fmax(kMinVarEI, var[c]));
      const double t = best_so_far - mu[c];
      const double ei = t * cdf(t / sigma) + sigma * pdf(t / sigma);
      values[c] = std::fmax(0.0, ei);
    }
    if (grads) {
      const double v = std::fmax(kMinVarGradEI, var[c]);
      const double sigma = std::sqrt(v);
      const double mu_diff = best_so_far - mu[c];
      const double C = mu_diff / sigma;
      const double pdf_C = pdf(C), cdf_C = cdf(C);
      for (int d = 0; d < dim; ++d) {
        const double gm = gmu[static_cast<size_t>(c) * dim + d];
        const double gchol = 0.5 * gvar[static_cast<size_t>(c) * dim + d] / sigma;
        const double d_C = (-sigma * gm - gchol * mu_diff) / v;
        const double d_A = -gm * cdf_C + mu_diff * pdf_C * d_C;
        const double d_B = gchol * pdf_C + sigma * (-C) * pdf_C * d_C;
        grads[static_cast<size_t>(c) * dim + d] = d_A + d_B;
      }
    }
  }
}

namespace {

// ---- the parallel axis inside the call: starts strided over several GPUs ---------------------------------------------
// (reference: OpenMP threads over starts, gpp_optimization.hpp:1472-1546).  One worker per device, each with its own
// bit-identical replica of the GP, its own plans and streams; one host thread per device and evaluation.
const cmoe_gp* replica_on(const cmoe_gp* gp, int device) {
  if (device == gp->device) return gp;
  if (gp->replicas_generation != gp->generation) {
    for (cmoe_gp* r : gp->replicas) cmoe_gp_destroy(r);
    gp->replicas.clear();
    gp->replicas_generation = gp->generation;
  }
  for (cmoe_gp* r : gp->replicas)
    if (r->device == device) return r;
  gp->replicas.push_back(clone_gp_to_device(gp, device));
  return gp->replicas.back();
}

struct DeviceWorker {
  const cmoe_gp* gp = nullptr;
  KgEvaluator kg;
  DevBuf<double> table;  // q-EI table on this device
  BatchEval eval;
  std::vector<double> pts, vals, grads;
  std::vector<int> idx;
};

struct ShardedEval {
  std::vector<std::unique_ptr<DeviceWorker>> workers;
  size_t ps = 0;
  void operator()(const double* pts, int nc, double* values, double* grads) {
    const int G = static_cast<int>(workers.size());
    if (G == 1) {
      workers[0]->eval(pts, nc, values, grads);
      return;
    }
    std::vector<std::exception_ptr> errs(G);
    std::vector<std::thread> threads;
    for (int d = 0; d < G; ++d) {
      DeviceWorker& w = *workers[d];
      w.idx.clear();
      for (int c = d; c < nc; c += G) w.idx.push_back(c);
      if (w.idx.empty()) continue;
      threads.emplace_back([&, d] {
        DeviceWorker& ww = *workers[d];
        try {
          const int m = static_cast<int>(ww.idx.size());
          ww.pts.resize(m * ps);
          ww.vals.resize(m);
          if (grads) ww.grads.resize(m * ps);
          for (int k = 0; k < m; ++k) std::copy(pts + ww.idx[k] * ps, pts + (ww.idx[k] + 1) * ps, ww.pts.begin() + k * ps);
          ww.eval(ww.pts.data(), m, ww.vals.data(), grads ? ww.grads.data() : nullptr);
        } catch (...) {
          errs[d] = std::current_exception();
        }
      });
    }
    for (auto& t : threads) t.join();
    for (int d = 0; d < G; ++d)
      if (errs[d]) std::rethrow_exception(errs[d]);
    for (int d = 0; d < G; ++d) {
      DeviceWorker& w = *workers[d];
      for (size_t k = 0; k < w.idx.size(); ++k) {
        values[w.idx[k]] = w.vals[k];
        if (grads) std::copy(w.grads.begin() + k * ps, w.grads.begin() + (k + 1) * ps, grads + w.idx[k] * ps);
      }
    }
  }
};

std::vector<int> device_list(const cmoe_gp* gp, const cmoe_multistart_opts* opts) {
  std::vector<int> devs;
  if (opts && opts->devices && opts->num_devices > 0) {
    const int count = cmoe_device_count();
    for (int i = 0; i < opts->num_devices; ++i) {
      CMOE_REQUIRE(opts->devices[i] >= 0 && opts->devices[i] < count, CMOE_ERR_BOUNDS, "device ordinal out of range");
      if (std::find(devs.begin(), devs.end(), opts->devices[i]) == devs.end()) devs.push_back(opts->devices[i]);
    }
  }
  if (devs.empty()) devs.push_back(gp->device);
  return devs;
}

// ---- ensembles of GPs ("MCMC-averaged" acquisition: one GP per hyper-parameter sample) -----------------------------
// KnowledgeGradientMCMCEvaluator (gpp_knowledge_gradient_mcmc_optimization.cpp:87-180): mean of the per-GP q-KG, divided
// by the fidelity cost max_i prod_{j >= dim-nf} x_ij, gradient by the quotient rule.
// ExpectedImprovementMCMCEvaluator (gpp_expected_improvement_mcmc_optimization.cpp:47-85): plain mean.
// Every GP sees the same normal draws (the reference hands one NormalRNG to every per-GP state and rewinds it per call).
// Divergence, documented in DESIGN.md: the reference's MCMC state refreshes only the FIRST candidate point in the copy
// it computes the cost from (..mcmc_optimization.cpp:187-188); the cost here always uses the current q points.
void apply_fidelity_cost(const double* pts, int nc, int q, int dim, int nf, int num_gp, double* values, double* grads) {
  const size_t ps = static_cast<size_t>(q) * dim;
  for (int c = 0; c < nc; ++c) {
    const double* x = pts + c * ps;
    double cost = 1.0;
    int index = -1;
    if (nf > 0) {
      cost = 0.0;
      for (int i = 0; i < q; ++i) {
        double point_cost = 1.0;
        for (int j = dim - nf; j < dim; ++j) point_cost *= x[static_cast<size_t>(i) * dim + j];
        if (cost < point_cost) {
          cost = point_cost;
          index = i;
        }
      }
    }
    const double kg_avg = values[c] / static_cast<double>(num_gp);
    values[c] = values[c] / (static_cast<double>(num_gp) * cost);
    if (grads) {
      double* g = grads + c * ps;
      for (size_t k = 0; k < ps; ++k) {
        double gradcost = 0.0;
        if (index >= 0 && k / dim == static_cast<size_t>(index) && static_cast<int>(k % dim) >= dim - nf)
          gradcost = cost / x[k];
        const double ga = g[k] / static_cast<double>(num_gp);
        g[k] = (ga * cost - kg_avg * gradcost) / (cost * cost);
      }
    }
  }
}

}  // namespace

void cmoe::check_ensemble(const cmoe_gp* const* gps, int num_gp) {
  CMOE_REQUIRE(gps != nullptr && num_gp >= 1, CMOE_ERR_BOUNDS, "an ensemble needs at least one GP");
  for (int m = 0; m < num_gp; ++m) {
    CMOE_REQUIRE(gps[m] != nullptr, CMOE_ERR_INVALID_VALUE, "NULL GP in ensemble");
    CMOE_REQUIRE(gps[m]->spec.dim == gps[0]->spec.dim && gps[m]->spec.g == gps[0]->spec.g &&
                     gps[m]->device == gps[0]->device,
                 CMOE_ERR_INVALID_VALUE, "ensemble members must share dim, derivative observations and device");
  }
}

cmoe::LargeUnionWork::~LargeUnionWork() {
  for (cudaEvent_t e : done) cudaEventDestroy(e);
}

cmoe::LargeUnionWork& cmoe::large_union_work(const cmoe_gp& gp, size_t bytes) {
  if (!gp.large_union_ws) gp.large_union_ws = std::make_shared<LargeUnionWork>();
  LargeUnionWork& w = *static_cast<LargeUnionWork*>(gp.large_union_ws.get());
  w.arena.ensure((bytes + sizeof(double) - 1) / sizeof(double));
  return w;
}

cmoe::MemberSchedule cmoe::schedule_members(int num_gp, int num_candidates, size_t avail, size_t per,
                                            size_t width_cap) {
  size_t width = std::min<size_t>({static_cast<size_t>(num_gp), avail / (per + kCarveSlack), width_cap});
  if (ensemble_members_in_flight() > 0) width = std::min<size_t>(width, ensemble_members_in_flight());
  width = std::max<size_t>(1, width);
  const size_t share = avail / width;
  const size_t chunk = chunk_items(num_candidates, share > kCarveSlack ? share - kCarveSlack : 0, per, kMaxChunkSets);
  return {static_cast<int>(width), static_cast<int>(chunk)};
}

void cmoe::run_members(const cmoe_gp* const* gps, int num_gp, int width, LargeUnionWork& ew,
                       const std::function<void(int, int)>& run) {
  while (ew.done.size() < static_cast<size_t>(num_gp)) {
    cudaEvent_t e;
    CMOE_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    ew.done.push_back(e);
  }
  // the members' streams are drained however the loop ends: the next evaluation reuses the region
  struct Drain {
    const cmoe_gp* const* gps;
    int n = 0;
    ~Drain() {
      for (int m = 0; m < n; ++m) cudaStreamSynchronize(gps[m]->stream);
    }
  } drain{gps};
  for (int m = 0; m < num_gp; ++m) {
    cudaStream_t s = gps[m]->stream;
    if (m >= width) CMOE_CUDA(cudaStreamWaitEvent(s, ew.done[m - width], 0));
    drain.n = m + 1;
    run(m, m % width);
    CMOE_CUDA(cudaEventRecord(ew.done[m], s));
  }
  drain.n = 0;
  for (int m = 0; m < num_gp; ++m) CMOE_CUDA(cudaStreamSynchronize(gps[m]->stream));
}

void cmoe::throw_singular_union(int minor) {
  throw Error(CMOE_ERR_SINGULAR,
              "GP-Variance matrix singular. Check for duplicate points_to_sample/being_sampled or "
              "points_to_sample/being_sampled duplicating points_sampled with 0 noise.",
              minor);
}

void cmoe::add_member(int m, int nc, size_t ps, const double* v, const double* g, double* values, double* grads) {
  if (m == 0) {
    std::copy(v, v + nc, values);
    if (grads) std::copy(g, g + nc * ps, grads);
    return;
  }
  for (int c = 0; c < nc; ++c) values[c] += v[c];
  if (grads)
    for (size_t k = 0; k < nc * ps; ++k) grads[k] += g[k];
}

void cmoe::drain_members(cudaStream_t s, int num_gp, int nc, size_t ps, const double* dval, const double* dgrad,
                         const int* dfail, double* values, double* grads) {
  const size_t all = static_cast<size_t>(num_gp) * nc;
  std::vector<int> f(all);
  std::vector<double> v(all), g(grads ? all * ps : 0);
  CMOE_CUDA(cudaMemcpyAsync(f.data(), dfail, all * sizeof(int), cudaMemcpyDeviceToHost, s));
  CMOE_CUDA(cudaMemcpyAsync(v.data(), dval, all * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (grads) CMOE_CUDA(cudaMemcpyAsync(g.data(), dgrad, all * ps * sizeof(double), cudaMemcpyDeviceToHost, s));
  CMOE_CUDA(cudaStreamSynchronize(s));
  for (size_t e = 0; e < all; ++e)
    if (f[e] != 0) throw_singular_union(f[e]);
  for (int m = 0; m < num_gp; ++m)
    add_member(m, nc, ps, v.data() + static_cast<size_t>(m) * nc, grads ? g.data() + m * nc * ps : nullptr, values,
               grads);
}

namespace {

// the mean of the members' sums
void ensemble_mean(int nc, size_t ps, int num_gp, double* values, double* grads) {
  for (int c = 0; c < nc; ++c) values[c] /= static_cast<double>(num_gp);
  if (grads)
    for (size_t k = 0; k < nc * ps; ++k) grads[k] /= static_cast<double>(num_gp);
}

// The q-EI evaluation of the drivers for an ensemble of num_gp >= 1 GPs: the mean of the members' q-EI.  With `analytic`
// and q = 1, p = 0 each member's is the closed-form one-point EI (gpp_math.hpp:1703-1749); otherwise the Monte-Carlo
// estimate on the normals of dtable (device [num_mc][q + p]) or Philox, per member on the per-set kernels up to kMaxQ
// union rows, past them one ei_large_eval call for every member.
BatchEval make_ei_eval(const cmoe_gp* const* gps_in, int num_gp, int q, const double* Xp_in, int p, int num_mc,
                       const double* best_in, uint64_t seed, bool analytic, const double* dtable) {
  const std::vector<const cmoe_gp*> gps(gps_in, gps_in + num_gp);
  const std::vector<double> best(best_in, best_in + num_gp);
  const int dim = gps[0]->spec.dim;
  const std::vector<double> Xp(Xp_in, Xp_in + static_cast<size_t>(p) * dim);
  const size_t ps = static_cast<size_t>(q) * dim;
  const bool closed_form = analytic && q == 1 && p == 0;
  if (!closed_form && ei_union_is_large(q, p)) {
    return [=](const double* pts, int nc, double* values, double* grads) {
      ei_large_eval(gps.data(), num_gp, pts, nc, q, Xp.data(), p, num_mc, best.data(), seed, dtable, values, grads);
      ensemble_mean(nc, ps, num_gp, values, grads);
    };
  }
  return [=](const double* pts, int nc, double* values, double* grads) {
    std::vector<double> tv(nc), tg(grads ? nc * ps : 0);
    for (int m = 0; m < num_gp; ++m) {
      if (closed_form) {
        analytic_ei(gps[m], pts, nc, best[m], tv.data(), grads ? tg.data() : nullptr);
      } else {
        require_device(gps[m]->device);  // may run on a worker thread of the multi-device driver
        ei_eval_batch(*gps[m], pts, nc, q, Xp.data(), p, num_mc, best[m], seed, dtable, tv.data(),
                      grads ? tg.data() : nullptr);
      }
      add_member(m, nc, ps, tv.data(), grads ? tg.data() : nullptr, values, grads);
    }
    ensemble_mean(nc, ps, num_gp, values, grads);
  };
}

// the MCMC drivers' q-EI: Monte-Carlo, or the closed form at q = 1, p = 0
BatchEval make_ei_ensemble(const cmoe_gp* const* gps, int num_gp, int q, const double* Xp, int p, int num_mc,
                           const double* best_so_far, uint64_t seed) {
  CMOE_REQUIRE(q >= 1 && p >= 0 && static_cast<long long>(q) + p <= kMaxSampleQ, CMOE_ERR_BOUNDS,
               "q + p must be in [1, 8192]");
  return make_ei_eval(gps, num_gp, q, Xp, p, num_mc, best_so_far, seed, true, nullptr);
}

// The MCMC drivers' q-KG: the members' sum divided by num_gp and the fidelity cost
BatchEval kg_ensemble_eval(KgEvaluator& ev, int q, int dim, int nf, int num_gp) {
  return [&ev, q, dim, nf, num_gp](const double* pts, int nc, double* values, double* grads) {
    ev(pts, nc, values, grads);
    apply_fidelity_cost(pts, nc, q, dim, nf, num_gp, values, grads);
  };
}

}  // namespace

void cmoe::validate_bounds(const double* b, int dim) {
  for (int d = 0; d < dim; ++d)
    CMOE_REQUIRE(b[2 * d] <= b[2 * d + 1], CMOE_ERR_BOUNDS, "Tensor product region is EMPTY.");
}

extern "C" {

int cmoe_limit_update(int domain_type, const double* domain_bounds, int dim, double max_relative_change,
                      const double* current_point, double* update) {
  return guarded(nullptr, [&] {
    CMOE_REQUIRE(dim >= 1 && dim <= CMOE_MAX_DIM, CMOE_ERR_BOUNDS, "dim must be in [1, CMOE_MAX_DIM]");
    if (domain_type == CMOE_DOMAIN_SIMPLEX) {
      limit_update_simplex_host(domain_bounds, dim, max_relative_change, current_point, update);
    } else {
      CMOE_REQUIRE(domain_type == CMOE_DOMAIN_TENSOR_PRODUCT, CMOE_ERR_INVALID_VALUE, "unknown domain type");
      for (int d = 0; d < dim; ++d)
        update[d] = limit_step(update[d], current_point[d], domain_bounds[2 * d], domain_bounds[2 * d + 1],
                                    max_relative_change);
    }
  });
}

int cmoe_multistart_kg_ex(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* outer, const cmoe_gd_params* inner,
                          const double* domain_bounds, const double* inner_bounds, const double* discrete_pts,
                          int num_pts, const double* starts, int num_starts, int q, const double* points_being_sampled,
                          int p, int num_mc, double best_so_far, uint64_t seed, const cmoe_multistart_opts* opts,
                          double* start_values, double* best_point, double* best_value, int* found_flag, int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(num_starts >= 1, CMOE_ERR_BOUNDS, "num_multistarts must be > 1");
    require_device(gp->device);
    validate_bounds(domain_bounds, gp->spec.dim);
    CMOE_REQUIRE(!opts || opts->domain_type == CMOE_DOMAIN_TENSOR_PRODUCT, CMOE_ERR_INVALID_VALUE,
                 "q-KG: only the tensor_product domain is implemented (the per-sample inner optimiser of the fused "
                 "kernel has no simplex LimitUpdate)");
    const std::vector<int> devs = device_list(gp, opts);
    const int G = static_cast<int>(devs.size());
    ShardedEval sh;
    sh.ps = static_cast<size_t>(q) * gp->spec.dim;
    for (int d = 0; d < G; ++d) {
      sh.workers.emplace_back(new DeviceWorker());
      DeviceWorker& w = *sh.workers.back();
      w.gp = replica_on(gp, devs[d]);
      // reference-driver behaviour: the discretisation set keeps the first start's points (cmoe_kg_plan_set_stale_union)
      const double* stale = (opts && opts->fresh_discretisation) ? nullptr
                            : (opts && opts->stale_union)        ? opts->stale_union
                                                                 : starts;
      make_kg_evaluator(w.kg, &w.gp, 1, num_fidelity, inner, inner_bounds, discrete_pts, num_pts, (num_starts + G - 1) / G,
                        (std::min(kTopK, num_starts) + G - 1) / G, q, points_being_sampled, p, num_mc, &best_so_far, seed,
                        stale);
      if (opts && opts->normals_table) w.kg.set_table(opts->normals_table, opts->table_len);
      w.eval = std::ref(w.kg);
    }
    BatchEval f = std::ref(sh);
    multistart_common(f, *outer, domain_bounds, q, gp->spec.dim, starts, num_starts,
                      -std::numeric_limits<double>::infinity(), start_values, best_point, best_value, found_flag);
    require_device(gp->device);
  });
}

int cmoe_multistart_kg(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* outer, const cmoe_gd_params* inner,
                       const double* domain_bounds, const double* inner_bounds, const double* discrete_pts, int num_pts,
                       const double* starts, int num_starts, int q, const double* points_being_sampled, int p,
                       int num_mc, double best_so_far, uint64_t seed, double* start_values, double* best_point,
                       double* best_value, int* found_flag, int* info) {
  return cmoe_multistart_kg_ex(gp, num_fidelity, outer, inner, domain_bounds, inner_bounds, discrete_pts, num_pts,
                               starts, num_starts, q, points_being_sampled, p, num_mc, best_so_far, seed, nullptr,
                               start_values, best_point, best_value, found_flag, info);
}

int cmoe_multistart_ei_ex(const cmoe_gp* gp, const cmoe_gd_params* outer, const double* domain_bounds,
                          const double* starts, int num_starts, int q, const double* points_being_sampled, int p,
                          int num_mc, double best_so_far, uint64_t seed, const cmoe_multistart_opts* opts,
                          double* start_values, double* best_point, double* best_value, int* found_flag, int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(num_starts >= 1, CMOE_ERR_BOUNDS, "num_multistarts must be > 1");
    require_device(gp->device);
    validate_bounds(domain_bounds, gp->spec.dim);
    const std::vector<int> devs = device_list(gp, opts);
    ShardedEval sh;
    sh.ps = static_cast<size_t>(q) * gp->spec.dim;
    const bool analytic = (q == 1 && p == 0);
    for (int dev : devs) {
      sh.workers.emplace_back(new DeviceWorker());
      DeviceWorker& w = *sh.workers.back();
      w.gp = replica_on(gp, dev);
      const double* dtable = nullptr;
      if (!analytic && opts && opts->normals_table) {
        CMOE_REQUIRE(opts->table_len >= static_cast<size_t>(num_mc) * (q + p), CMOE_ERR_INVALID_VALUE,
                     "All random numbers stored in the RNG have been used up!");
        require_device(dev);
        w.table.upload(opts->normals_table, opts->table_len, w.gp->stream);
        CMOE_CUDA(cudaStreamSynchronize(w.gp->stream));
        dtable = w.table.p;
      }
      w.eval = make_ei_eval(&w.gp, 1, q, points_being_sampled, p, num_mc, &best_so_far, seed, true, dtable);
    }
    BatchEval f = std::ref(sh);
    const int domain_type = opts ? opts->domain_type : CMOE_DOMAIN_TENSOR_PRODUCT;
    CMOE_REQUIRE(domain_type == CMOE_DOMAIN_TENSOR_PRODUCT || domain_type == CMOE_DOMAIN_SIMPLEX, CMOE_ERR_INVALID_VALUE,
                 "unknown domain type");
    multistart_common(f, *outer, domain_bounds, q, gp->spec.dim, starts, num_starts, -1.0, start_values, best_point,
                      best_value, found_flag, domain_type);
    require_device(gp->device);
  });
}

int cmoe_multistart_ei(const cmoe_gp* gp, const cmoe_gd_params* outer, const double* domain_bounds,
                       const double* starts, int num_starts, int q, const double* points_being_sampled, int p,
                       int num_mc, double best_so_far, uint64_t seed, double* start_values, double* best_point,
                       double* best_value, int* found_flag, int* info) {
  return cmoe_multistart_ei_ex(gp, outer, domain_bounds, starts, num_starts, q, points_being_sampled, p, num_mc,
                               best_so_far, seed, nullptr, start_values, best_point, best_value, found_flag, info);
}

int cmoe_kg_gradient_descent_ex(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* outer,
                                const cmoe_gd_params* inner, const double* domain_bounds, const double* inner_bounds,
                                const double* discrete_pts, int num_pts, const double* starts, int num_starts, int q,
                                const double* points_being_sampled, int p, int num_mc, double best_so_far,
                                uint64_t seed, const double* stale_union, double* values_out, double* points_out,
                                int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(num_starts >= 1, CMOE_ERR_BOUNDS, "num_multistarts must be > 1");
    require_device(gp->device);
    validate_bounds(domain_bounds, gp->spec.dim);
    KgEvaluator ev;
    make_kg_evaluator(ev, &gp, 1, num_fidelity, inner, inner_bounds, discrete_pts, num_pts, num_starts, num_starts, q,
                      points_being_sampled, p, num_mc, &best_so_far, seed, stale_union);
    BatchEval f = std::ref(ev);
    gradient_descent_batch(f, *outer, domain_bounds, q, gp->spec.dim, starts, num_starts, values_out, points_out);
  });
}

int cmoe_kg_gradient_descent(const cmoe_gp* gp, int num_fidelity, const cmoe_gd_params* outer,
                             const cmoe_gd_params* inner, const double* domain_bounds, const double* inner_bounds,
                             const double* discrete_pts, int num_pts, const double* starts, int num_starts, int q,
                             const double* points_being_sampled, int p, int num_mc, double best_so_far, uint64_t seed,
                             double* values_out, double* points_out, int* info) {
  return cmoe_kg_gradient_descent_ex(gp, num_fidelity, outer, inner, domain_bounds, inner_bounds, discrete_pts, num_pts,
                                     starts, num_starts, q, points_being_sampled, p, num_mc, best_so_far, seed, nullptr,
                                     values_out, points_out, info);
}

int cmoe_ei_gradient_descent(const cmoe_gp* gp, const cmoe_gd_params* outer, const double* domain_bounds,
                             const double* starts, int num_starts, int q, const double* points_being_sampled, int p,
                             int num_mc, double best_so_far, uint64_t seed, double* values_out, double* points_out,
                             int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(num_starts >= 1, CMOE_ERR_BOUNDS, "num_multistarts must be > 1");
    require_device(gp->device);
    validate_bounds(domain_bounds, gp->spec.dim);
    BatchEval f = make_ei_eval(&gp, 1, q, points_being_sampled, p, num_mc, &best_so_far, seed, true, nullptr);
    gradient_descent_batch(f, *outer, domain_bounds, q, gp->spec.dim, starts, num_starts, values_out, points_out);
  });
}

int cmoe_kg_eval_mcmc(const cmoe_gp* const* gps, int num_gp, int num_fidelity, const cmoe_gd_params* inner,
                      const double* inner_bounds, const double* discrete_pts, int num_pts, const double* candidates,
                      int num_candidates, int q, const double* points_being_sampled, int p, int num_mc,
                      const double* best_so_far, uint64_t seed, const double* normals_table, double* values,
                      double* grads, int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(static_cast<long long>(q) + p <= CMOE_MAX_KG_LARGE_ROWS, CMOE_ERR_BOUNDS,
                 "(q+p)*(1+num_derivatives) must be <= 1024");
    check_ensemble(gps, num_gp);
    CMOE_REQUIRE(num_candidates >= 1, CMOE_ERR_BOUNDS, "num_multistarts must be > 1");
    const int dim = gps[0]->spec.dim;
    const size_t ps = static_cast<size_t>(q) * dim;
    if (kg_union_is_large(q, p, gps[0]->spec.g)) {
      kg_large_eval(gps, num_gp, num_fidelity, inner, inner_bounds, discrete_pts, num_pts, candidates, num_candidates,
                    q, points_being_sampled, p, num_mc, best_so_far, seed, normals_table, nullptr, values, grads,
                    nullptr);
    } else {
      // each member's cmoe_kg_eval, which reuses its handle's cached plan across calls
      std::vector<double> tv(num_candidates), tg(grads ? num_candidates * ps : 0);
      for (int m = 0; m < num_gp; ++m) {
        int inf = 0;
        const int rc = cmoe_kg_eval(gps[m], num_fidelity, inner, inner_bounds,
                                    discrete_pts + static_cast<size_t>(m) * num_pts * (dim - num_fidelity), num_pts,
                                    candidates, num_candidates, q, points_being_sampled, p, num_mc, best_so_far[m],
                                    seed, normals_table, tv.data(), grads ? tg.data() : nullptr, nullptr, &inf);
        if (rc != CMOE_OK) throw Error(rc, cmoe_last_error(), inf);
        add_member(m, num_candidates, ps, tv.data(), grads ? tg.data() : nullptr, values, grads);
      }
    }
    apply_fidelity_cost(candidates, num_candidates, q, dim, num_fidelity, num_gp, values, grads);
  });
}

int cmoe_ei_analytic(const cmoe_gp* gp, const double* points, int num_points, double best_so_far, double* values,
                     double* grads, int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(num_points >= 1, CMOE_ERR_BOUNDS, "num_multistarts must be > 1");
    require_device(gp->device);
    analytic_ei(gp, points, num_points, best_so_far, values, grads);
  });
}

int cmoe_ei_eval_mcmc(const cmoe_gp* const* gps, int num_gp, const double* candidates, int num_candidates, int q,
                      const double* points_being_sampled, int p, int num_mc, const double* best_so_far, uint64_t seed,
                      const double* normals_table, int analytic_single, double* values, double* grads, int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(static_cast<long long>(q) + p <= kMaxSampleQ, CMOE_ERR_BOUNDS, "q + p must be <= 8192");
    check_ensemble(gps, num_gp);
    CMOE_REQUIRE(num_candidates >= 1, CMOE_ERR_BOUNDS, "num_multistarts must be > 1");
    require_device(gps[0]->device);
    // the kernels read the table from device memory: a host pointer is only readable by the GPU where the system
    // maps pageable host memory for it, and faults elsewhere
    DevBuf<double> dtable;
    if (normals_table) {
      dtable.upload(normals_table, static_cast<size_t>(num_mc) * (q + p), gps[0]->stream);
      CMOE_CUDA(cudaStreamSynchronize(gps[0]->stream));  // the members evaluate on their own streams
    }
    make_ei_eval(gps, num_gp, q, points_being_sampled, p, num_mc, best_so_far, seed, analytic_single != 0,
                 normals_table ? dtable.p : nullptr)(candidates, num_candidates, values, grads);
  });
}

int cmoe_multistart_kg_mcmc(const cmoe_gp* const* gps, int num_gp, int num_fidelity, const cmoe_gd_params* outer,
                            const cmoe_gd_params* inner, const double* domain_bounds, const double* inner_bounds,
                            const double* discrete_pts, int num_pts, const double* starts, int num_starts, int q,
                            const double* points_being_sampled, int p, int num_mc, const double* best_so_far,
                            uint64_t seed, double* start_values, double* best_point, double* best_value,
                            int* found_flag, int* info) {
  return guarded(info, [&] {
    check_ensemble(gps, num_gp);
    CMOE_REQUIRE(num_starts >= 1, CMOE_ERR_BOUNDS, "num_multistarts must be > 1");
    require_device(gps[0]->device);
    validate_bounds(domain_bounds, gps[0]->spec.dim);
    KgEvaluator ev;
    make_kg_evaluator(ev, gps, num_gp, num_fidelity, inner, inner_bounds, discrete_pts, num_pts, num_starts,
                      std::min(kTopK, num_starts), q, points_being_sampled, p, num_mc, best_so_far, seed);
    BatchEval f = kg_ensemble_eval(ev, q, gps[0]->spec.dim, num_fidelity, num_gp);
    multistart_common(f, *outer, domain_bounds, q, gps[0]->spec.dim, starts, num_starts,
                      -std::numeric_limits<double>::infinity(), start_values, best_point, best_value, found_flag);
  });
}

int cmoe_multistart_ei_mcmc(const cmoe_gp* const* gps, int num_gp, const cmoe_gd_params* outer,
                            const double* domain_bounds, const double* starts, int num_starts, int q,
                            const double* points_being_sampled, int p, int num_mc, const double* best_so_far,
                            uint64_t seed, double* start_values, double* best_point, double* best_value,
                            int* found_flag, int* info) {
  return guarded(info, [&] {
    check_ensemble(gps, num_gp);
    CMOE_REQUIRE(num_starts >= 1, CMOE_ERR_BOUNDS, "num_multistarts must be > 1");
    require_device(gps[0]->device);
    validate_bounds(domain_bounds, gps[0]->spec.dim);
    BatchEval f = make_ei_ensemble(gps, num_gp, q, points_being_sampled, p, num_mc, best_so_far, seed);
    // io_container starts from 0.0 in the MCMC drivers (gpp_expected_improvement_mcmc_optimization.hpp:914,968)
    multistart_common(f, *outer, domain_bounds, q, gps[0]->spec.dim, starts, num_starts, 0.0, start_values, best_point,
                      best_value, found_flag);
  });
}

int cmoe_kg_gradient_descent_mcmc(const cmoe_gp* const* gps, int num_gp, int num_fidelity, const cmoe_gd_params* outer,
                                  const cmoe_gd_params* inner, const double* domain_bounds, const double* inner_bounds,
                                  const double* discrete_pts, int num_pts, const double* starts, int num_starts, int q,
                                  const double* points_being_sampled, int p, int num_mc, const double* best_so_far,
                                  uint64_t seed, double* values_out, double* points_out, int* info) {
  return guarded(info, [&] {
    check_ensemble(gps, num_gp);
    CMOE_REQUIRE(num_starts >= 1, CMOE_ERR_BOUNDS, "num_multistarts must be > 1");
    require_device(gps[0]->device);
    validate_bounds(domain_bounds, gps[0]->spec.dim);
    KgEvaluator ev;
    make_kg_evaluator(ev, gps, num_gp, num_fidelity, inner, inner_bounds, discrete_pts, num_pts, num_starts, num_starts,
                      q, points_being_sampled, p, num_mc, best_so_far, seed);
    BatchEval f = kg_ensemble_eval(ev, q, gps[0]->spec.dim, num_fidelity, num_gp);
    gradient_descent_batch(f, *outer, domain_bounds, q, gps[0]->spec.dim, starts, num_starts, values_out, points_out);
  });
}

int cmoe_ei_gradient_descent_mcmc(const cmoe_gp* const* gps, int num_gp, const cmoe_gd_params* outer,
                                  const double* domain_bounds, const double* starts, int num_starts, int q,
                                  const double* points_being_sampled, int p, int num_mc, const double* best_so_far,
                                  uint64_t seed, double* values_out, double* points_out, int* info) {
  return guarded(info, [&] {
    check_ensemble(gps, num_gp);
    CMOE_REQUIRE(num_starts >= 1, CMOE_ERR_BOUNDS, "num_multistarts must be > 1");
    require_device(gps[0]->device);
    validate_bounds(domain_bounds, gps[0]->spec.dim);
    BatchEval f = make_ei_ensemble(gps, num_gp, q, points_being_sampled, p, num_mc, best_so_far, seed);
    gradient_descent_batch(f, *outer, domain_bounds, q, gps[0]->spec.dim, starts, num_starts, values_out, points_out);
  });
}

// MultistartGradientDescentHyperparameterOptimization (gpp_model_selection.hpp:1063-1103) with one thread: the best
// start by InitializeBestKnownPoint (:911-930), then GradientDescentOptimizer::Optimize from EVERY start (no top-20
// screening), then the arg-max of MultistartOptimize (gpp_optimization.hpp:1504-1545).  The point is the set itself,
// so the descent runs on one "point" of nh coordinates over the linear-space box.
int cmoe_hyperparameter_gradient_descent(int kernel, const cmoe_gd_params* gd_params, const double* bounds,
                                         const double* starts, int num_starts, const double* points_sampled,
                                         const double* points_sampled_value, const int* derivatives,
                                         int num_derivatives, int dim, int num_sampled, int device,
                                         double* best_point, double* best_value, int* found_flag,
                                         double* end_points, double* end_values, int* info) {
  return guarded(info, [&] {
    CMOE_REQUIRE(num_starts >= 1, CMOE_ERR_BOUNDS, "num_multistarts must be > 1");
    CMOE_REQUIRE(gd_params != nullptr && bounds != nullptr && starts != nullptr && best_point != nullptr,
                 CMOE_ERR_INVALID_VALUE, "NULL argument");
    CMOE_REQUIRE(dim >= 1 && dim <= CMOE_MAX_DIM, CMOE_ERR_BOUNDS, "dim must be in [1, CMOE_MAX_DIM]");
    CMOE_REQUIRE(num_derivatives >= 0 && num_derivatives <= dim, CMOE_ERR_BOUNDS, "num_derivatives out of range");
    const int nh = 2 + dim + num_derivatives;
    validate_bounds(bounds, nh);
    BatchEval eval = [&](const double* pts, int nc, double* values, double* grads) {
      int linfo = 0;
      const int rc = grads ? cmoe_grad_log_marginal_likelihood_list(kernel, pts, nc, points_sampled,
                                                                    points_sampled_value, derivatives, num_derivatives,
                                                                    dim, num_sampled, device, values, grads, &linfo)
                           : cmoe_log_marginal_likelihood_list(kernel, pts, nc, points_sampled, points_sampled_value,
                                                               derivatives, num_derivatives, dim, num_sampled, device,
                                                               values, &linfo);
      if (rc != CMOE_OK) throw Error(rc, cmoe_last_error(), linfo);
    };
    std::vector<double> start_v(num_starts), fin_v(num_starts), fin_p(static_cast<size_t>(num_starts) * nh);
    eval(starts, num_starts, start_v.data(), nullptr);
    // InitializeBestKnownPoint: -inf and the first start, strict `<`
    double init_best = -std::numeric_limits<double>::infinity();
    int ib = 0;
    for (int i = 0; i < num_starts; ++i)
      if (init_best < start_v[i]) {
        init_best = start_v[i];
        ib = i;
      }
    gradient_descent_batch(eval, *gd_params, bounds, 1, nh, starts, num_starts, fin_v.data(), fin_p.data());
    // MultistartOptimize: the running best starts at init_best; an end value replaces it only if strictly larger
    double best = init_best;
    int bi = -1;
    for (int i = 0; i < num_starts; ++i)
      if (best < fin_v[i]) {
        best = fin_v[i];
        bi = i;
      }
    const double* bp = (bi >= 0) ? fin_p.data() + static_cast<size_t>(bi) * nh : starts + static_cast<size_t>(ib) * nh;
    std::copy(bp, bp + nh, best_point);
    if (best_value) *best_value = best;
    if (found_flag) *found_flag = bi >= 0 ? 1 : 0;
    if (end_points) std::copy(fin_p.begin(), fin_p.end(), end_points);
    if (end_values) std::copy(fin_v.begin(), fin_v.end(), end_values);
  });
}

}  // extern "C"
