// Autotuner: Bayesian optimisation (Gaussian process + expected improvement)
// of continuous engine knobs, plus sequential search over categorical ones.
//
// Parity: horovod/common/parameter_manager.{h,cc} (joint fusion-threshold ×
// cycle-time Bayesian search with 4 seed points then EI up to 20 samples,
// noise α = 0.8, categorical knobs tried sequentially, score = median of 5
// samples of bytes/µs — parameter_manager.cc:28-31,45-56,155-181,391-402,
// 462-475) and horovod/common/optim/{bayesian_optimization,gaussian_process}.cc
// (Eigen + L-BFGS there; a dense Cholesky and random-restart EI search here —
// the problem is ≤ 4-D with ≤ 24 samples).  What is tuned: comm-kernel
// CTA count, sparse-kernel CTA cap, bucket size, one-shot/two-shot threshold.
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <random>
#include <unordered_map>
#include <vector>

namespace {

struct Tuner {
  int nd = 0;
  std::vector<double> lo, hi;
  std::vector<std::vector<double>> X;   // normalised samples
  std::vector<double> y;                // scores (higher is better)
  std::vector<double> pending;          // last suggestion (normalised)
  std::vector<double> samples;          // raw samples for the pending point
  int samples_per_point = 5;
  int max_points = 20;
  int warmups = 3, seen = 0;
  double alpha = 0.8, length = 0.3;
  std::mt19937 rng{12345};
  bool done = false;
  // categorical knobs: value index per knob, tried sequentially after the joint search
  std::vector<int> cat_sizes, cat_best, cat_cur;
  std::vector<double> cat_best_score;
  int cat_knob = -1;
  double best_score = -1e300;
  std::vector<double> best_x;
};

std::mutex g_mu;
std::unordered_map<int, Tuner*> g_tuners;
int g_next = 1;

double kern(const Tuner& t, const std::vector<double>& a, const std::vector<double>& b) {
  double d2 = 0;
  for (int i = 0; i < t.nd; ++i) d2 += (a[i] - b[i]) * (a[i] - b[i]);
  return std::exp(-0.5 * d2 / (t.length * t.length));
}

// Cholesky of K (n×n, row-major) in place; returns false if not PD
bool chol(std::vector<double>& K, int n) {
  for (int j = 0; j < n; ++j) {
    double s = K[j * n + j];
    for (int k = 0; k < j; ++k) s -= K[j * n + k] * K[j * n + k];
    if (s <= 1e-12) return false;
    K[j * n + j] = std::sqrt(s);
    for (int i = j + 1; i < n; ++i) {
      double v = K[i * n + j];
      for (int k = 0; k < j; ++k) v -= K[i * n + k] * K[j * n + k];
      K[i * n + j] = v / K[j * n + j];
    }
  }
  return true;
}
void solve_lower(const std::vector<double>& L, int n, std::vector<double>& b) {
  for (int i = 0; i < n; ++i) {
    double v = b[i];
    for (int k = 0; k < i; ++k) v -= L[i * n + k] * b[k];
    b[i] = v / L[i * n + i];
  }
}
void solve_upper_t(const std::vector<double>& L, int n, std::vector<double>& b) {
  for (int i = n - 1; i >= 0; --i) {
    double v = b[i];
    for (int k = i + 1; k < n; ++k) v -= L[k * n + i] * b[k];
    b[i] = v / L[i * n + i];
  }
}

double norm_pdf(double z) { return std::exp(-0.5 * z * z) / std::sqrt(2 * M_PI); }
double norm_cdf(double z) { return 0.5 * std::erfc(-z / std::sqrt(2.0)); }

std::vector<double> next_point(Tuner& t) {
  static const double seeds[4][2] = {{0.0625, 0.05}, {0.5, 0.5}, {0.25, 0.25}, {0.125, 0.1}};
  const int n = (int)t.X.size();
  std::vector<double> x(t.nd, 0.5);
  if (n < 4) {
    for (int i = 0; i < t.nd; ++i) x[i] = seeds[n][i % 2];
    return x;
  }
  // normalise scores
  double mean = 0, sd = 0;
  for (double v : t.y) mean += v;
  mean /= n;
  for (double v : t.y) sd += (v - mean) * (v - mean);
  sd = std::sqrt(sd / n) + 1e-9;
  std::vector<double> yn(n);
  for (int i = 0; i < n; ++i) yn[i] = (t.y[i] - mean) / sd;
  std::vector<double> K(n * n);
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < n; ++j) K[i * n + j] = kern(t, t.X[i], t.X[j]) + (i == j ? t.alpha * t.alpha * 0.1 : 0);
  if (!chol(K, n)) { for (int i = 0; i < t.nd; ++i) x[i] = std::uniform_real_distribution<>(0, 1)(t.rng); return x; }
  std::vector<double> a = yn;
  solve_lower(K, n, a);
  solve_upper_t(K, n, a);
  const double ybest = *std::max_element(yn.begin(), yn.end());
  double best_ei = -1;
  std::uniform_real_distribution<> U(0, 1);
  for (int c = 0; c < 2000; ++c) {
    std::vector<double> cand(t.nd);
    for (int i = 0; i < t.nd; ++i) cand[i] = U(t.rng);
    std::vector<double> ks(n);
    for (int i = 0; i < n; ++i) ks[i] = kern(t, cand, t.X[i]);
    double mu = 0;
    for (int i = 0; i < n; ++i) mu += ks[i] * a[i];
    std::vector<double> v = ks;
    solve_lower(K, n, v);
    double var = 1.0;
    for (int i = 0; i < n; ++i) var -= v[i] * v[i];
    const double s = std::sqrt(std::max(var, 1e-12));
    const double z = (mu - ybest - 0.01) / s;
    const double ei = (mu - ybest - 0.01) * norm_cdf(z) + s * norm_pdf(z);
    if (ei > best_ei) { best_ei = ei; x = cand; }
  }
  return x;
}

}  // namespace

extern "C" {

int px_autotune_create(int nd, const double* lo, const double* hi, int n_cat, const int* cat_sizes,
                       int samples_per_point, int max_points, int warmups, unsigned seed) {
  Tuner* t = new Tuner();
  t->nd = nd; t->lo.assign(lo, lo + nd); t->hi.assign(hi, hi + nd);
  t->samples_per_point = samples_per_point > 0 ? samples_per_point : 5;
  t->max_points = max_points > 0 ? max_points : 20;
  t->warmups = warmups >= 0 ? warmups : 3;
  t->rng.seed(seed ? seed : 12345);
  for (int i = 0; i < n_cat; ++i) {
    t->cat_sizes.push_back(cat_sizes[i]); t->cat_best.push_back(0); t->cat_cur.push_back(0);
    t->cat_best_score.push_back(-1e300);
  }
  t->pending = next_point(*t);
  std::lock_guard<std::mutex> lk(g_mu);
  g_tuners[g_next] = t;
  return g_next++;
}

// current parameters to run with: x[nd] (de-normalised) and cat[n_cat]
int px_autotune_current(int h, double* x, int* cat) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_tuners.find(h);
  if (it == g_tuners.end()) return -1;
  Tuner& t = *it->second;
  const std::vector<double>& p = (t.done || t.cat_knob >= 0) && !t.best_x.empty() ? t.best_x : t.pending;
  for (int i = 0; i < t.nd; ++i) x[i] = t.lo[i] + p[i] * (t.hi[i] - t.lo[i]);
  for (size_t i = 0; i < t.cat_sizes.size(); ++i) cat[i] = t.done ? t.cat_best[i] : t.cat_cur[i];
  return t.done ? 1 : 0;
}

// feed one throughput sample (e.g. bytes/µs or items/s) measured with the
// current parameters; returns 1 when the parameters changed, 2 when finished
int px_autotune_report(int h, double score) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_tuners.find(h);
  if (it == g_tuners.end()) return -1;
  Tuner& t = *it->second;
  if (t.done) return 2;
  if (t.seen < t.warmups) { t.seen++; return 0; }
  t.samples.push_back(score);
  if ((int)t.samples.size() < t.samples_per_point) return 0;
  std::sort(t.samples.begin(), t.samples.end());
  const double med = t.samples[t.samples.size() / 2];
  t.samples.clear();
  t.seen = 0;
  if (t.cat_knob < 0) {             // joint continuous search
    t.X.push_back(t.pending); t.y.push_back(med);
    if (med > t.best_score) { t.best_score = med; t.best_x = t.pending; }
    if ((int)t.X.size() >= t.max_points || t.nd == 0) {
      t.cat_knob = 0;
      if (t.cat_sizes.empty()) { t.done = true; return 2; }
      t.cat_cur = t.cat_best; t.cat_cur[0] = 0;
    } else t.pending = next_point(t);
    return 1;
  }
  // categorical: sequential sweep of knob `cat_knob`
  const int k = t.cat_knob;
  if (med > t.cat_best_score[k]) { t.cat_best_score[k] = med; t.cat_best[k] = t.cat_cur[k]; }
  if (t.cat_cur[k] + 1 < t.cat_sizes[k]) { t.cat_cur[k]++; return 1; }
  t.cat_cur[k] = t.cat_best[k];
  t.cat_knob++;
  if (t.cat_knob >= (int)t.cat_sizes.size()) { t.done = true; return 2; }
  t.cat_cur[t.cat_knob] = 0;
  return 1;
}

int px_autotune_num_points(int h) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_tuners.find(h);
  return it == g_tuners.end() ? -1 : (int)it->second->X.size();
}

double px_autotune_best_score(int h) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_tuners.find(h);
  return it == g_tuners.end() ? 0 : it->second->best_score;
}

int px_autotune_destroy(int h) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_tuners.find(h);
  if (it == g_tuners.end()) return -1;
  delete it->second; g_tuners.erase(it);
  return 0;
}

}  // extern "C"
