// bsb_score: bsuite scores of every lane from the log rows, in one launch for the whole suite (plus a tiny tag pass).
// The per-experiment rules are the __host__ __device__ functions of bsb_score.cuh; this file holds the constants,
// the kernels, the host loop and the C entry point.
#include <algorithm>
#include <cstring>
#include <mutex>
#include <vector>

#include "bsb_env.h"
#include "bsb_score.cuh"

using namespace bsb;

namespace {

// One entry per experiment, in sorted name order (enum bsb_experiment).  NUM_EPISODES and TAGS restate
// experiments/<name>/sweep.py; the constants are those of experiments/<name>/analysis.py.
const ExperimentScoring kScoring[NUM_EXPERIMENTS] = {
    {SK_REGRET, 0, 10000, T_BASIC, 0.5, 0., 0.},                                   // bandit/analysis.py:27, 31-34
    {SK_REGRET, 1, 10000, T_NOISE, 0.5, 0., 0.},                                   // bandit_noise/analysis.py:31-37
    {SK_REGRET, 1, 10000, T_SCALE, 0.5, 0., 0.},                                   // bandit_scale/analysis.py:31-32
    {SK_CARTPOLE, 0, 1000, T_BASIC | T_CREDIT | T_GENERALIZATION, 1000., 0., 0.},  // cartpole/analysis.py:27-50
    {SK_CARTPOLE, 1, 1000, T_NOISE | T_GENERALIZATION, 1000., 0., 0.},            // cartpole_noise/analysis.py:31-37
    {SK_CARTPOLE, 1, 1000, T_SCALE | T_GENERALIZATION, 1000., 0., 0.},            // cartpole_scale/analysis.py:30-31
    {SK_SWINGUP, 0, 1000, T_EXPLORATION | T_GENERALIZATION, 700., 0., 0.},        // cartpole_swingup/analysis.py:27-54
    {SK_REGRET, 0, 10000, T_BASIC | T_CREDIT, 1.6, 0., 0.},                        // catch/analysis.py:26, 30-33
    {SK_REGRET, 1, 10000, T_NOISE | T_CREDIT, 1.6, 0., 0.},                        // catch_noise/analysis.py:31-37
    {SK_REGRET, 1, 10000, T_SCALE | T_CREDIT, 1.6, 0., 0.},                        // catch_scale/analysis.py:30-31
    {SK_DEEP_SEA, 0, 10000, T_EXPLORATION, 0., 0.9, 0.},                           // deep_sea/analysis.py:37-91
    {SK_DEEP_SEA, 0, 10000, T_EXPLORATION | T_NOISE, 0., 0.8, 100.},              // deep_sea_stochastic/analysis.py:42-58
    {SK_DISCOUNTING, 0, 1000, T_CREDIT, 0., 0., 0.},                               // discounting_chain/analysis.py:33-38
    {SK_MEMORY, 0, 10000, T_MEMORY, 0., 0.75, 0.},                                 // memory_len/analysis.py:28-51
    {SK_MEMORY, 0, 10000, T_MEMORY, 0., 0.75, 0.},                                 // memory_size/analysis.py:29-30
    {SK_MNIST, 0, 10000, T_BASIC | T_GENERALIZATION, 1.8, 0., 0.},                // mnist/analysis.py:27, 31-42
    {SK_MNIST, 1, 10000, T_NOISE | T_GENERALIZATION, 1.8, 0., 0.},                // mnist_noise/analysis.py:30-36
    {SK_MNIST, 1, 10000, T_SCALE | T_GENERALIZATION, 1.8, 0., 0.},                // mnist_scale/analysis.py:30-31
    {SK_MOUNTAIN_CAR, 0, 1000, T_BASIC | T_GENERALIZATION, 1000., 0., 0.},        // mountain_car/analysis.py:25-44
    {SK_MOUNTAIN_CAR, 1, 1000, T_NOISE | T_GENERALIZATION, 1000., 0., 0.},        // mountain_car_noise/analysis.py:31-37
    {SK_MOUNTAIN_CAR, 1, 1000, T_SCALE | T_GENERALIZATION, 1000., 0., 0.},        // mountain_car_scale/analysis.py:30-31
    {SK_UMBRELLA, 0, 10000, T_CREDIT | T_NOISE, 0., 0.5, 0.},                      // umbrella_distract/analysis.py:30-31
    {SK_UMBRELLA, 0, 10000, T_CREDIT | T_NOISE, 0., 0.5, 0.},                      // umbrella_length/analysis.py:28-44
};

constexpr int kScoreThreads = 128;

// Everything a launch reads besides the rows, passed by value (about 25 KB of kernel parameters, so a call needs no
// device allocation and a second call cannot overwrite what a queued one still has to read).
struct ScoreJob {
  int64_t lanes;
  int32_t begin[NUM_EXPERIMENTS + 1];     // sources of experiment e: [begin[e], begin[e + 1])
  ExperimentScoring x[NUM_EXPERIMENTS];
  ScoreSrc src[BSB_SCORE_MAX_SOURCES];
};

// summary_analysis.py:149-171 (_summarize_single_by_tag, ave_score_by_tag) for lane j: per tag the pandas mean of
// the scores of the tagged experiments present, in sorted name order.
BSB_HD void tag_means(const ScoreJob& job, const double* scores, int64_t j, double* tag_scores) {
  for (int t = 0; t < NUM_TAGS; ++t) {
    SkipNaNMean m;
    for (int e = 0; e < NUM_EXPERIMENTS; ++e) {
      if (!(job.x[e].tags & (1 << t))) continue;
      const double s = scores[(int64_t)e * job.lanes + j];
      if (s == s || experiment_present(job.src + job.begin[e], job.begin[e + 1] - job.begin[e], j)) m.add(s);
    }
    tag_scores[(int64_t)t * job.lanes + j] = m.mean();
  }
}

}  // namespace

__global__ void __launch_bounds__(kScoreThreads) score_kernel(const __grid_constant__ ScoreJob job, double* scores,
                                                               uint8_t* finished) {
  const int e = blockIdx.y;
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= job.lanes) return;
  double s;
  bool f;
  score_experiment(job.src + job.begin[e], job.begin[e + 1] - job.begin[e], job.x[e], j, &s, &f);
  scores[(int64_t)e * job.lanes + j] = s;
  finished[(int64_t)e * job.lanes + j] = f ? 1 : 0;
}

__global__ void __launch_bounds__(kScoreThreads) score_tags_kernel(const __grid_constant__ ScoreJob job,
                                                                    const double* scores, double* tag_scores) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < job.lanes) tag_means(job, scores, j, tag_scores);
}

namespace {

struct DeviceScope {
  int prev; bool on;
  explicit DeviceScope(int dev) : prev(0), on(dev >= 0) { if (on) { cudaGetDevice(&prev); cudaSetDevice(dev); } }
  ~DeviceScope() { if (on) cudaSetDevice(prev); }
};

struct Resolved { ScoreSrc src; int experiment, setting, device; };

// Checks one source and turns it into the scorer's view of its rows.
int resolve(const bsb_score_source& in, int64_t lanes, Resolved* out) {
  if (in.experiment < 0 || in.experiment >= NUM_EXPERIMENTS) return fail(BSB_INVALID_ARGUMENT, "unknown experiment");
  if (in.setting < 0) return fail(BSB_INVALID_ARGUMENT, "setting must be >= 0");
  const double* rows;
  const int32_t* counts;
  int64_t n_points, n_columns, stride;
  int device;
  if (in.env) {
    bsb_env* env = in.env;
    if (!env->p.log_rows) return fail(BSB_INVALID_ARGUMENT, "environment was created without a log schedule");
    { int frc = drain_log_rows(env); if (frc != BSB_OK) return frc; }
    rows = env->p.log_rows; counts = env->p.log_next;
    n_points = env->p.n_log_points; n_columns = 5 + env->names.n; stride = env->p.batch; device = env->device;
  } else {
    if (!in.rows || !in.counts) return fail(BSB_INVALID_ARGUMENT, "a source needs a handle or rows and counts");
    rows = in.rows; counts = in.counts;
    n_points = in.n_points; n_columns = in.n_columns; stride = in.lane_stride; device = in.device;
    if (n_points < 0 || n_points > 4096) return fail(BSB_INVALID_ARGUMENT, "n_points must be in [0, 4096]");
    if (n_columns < 1 || n_columns > 5 + BSB_MAX_INFO) return fail(BSB_INVALID_ARGUMENT, "n_columns out of range");
    if (device < 0 && device != BSB_DEVICE_HOST) return fail(BSB_INVALID_ARGUMENT, "device must be >= 0 or BSB_DEVICE_HOST");
  }
  if (in.lanes != lanes) return fail(BSB_INVALID_ARGUMENT, "sources have different lane counts");
  if (in.first_lane < 0 || in.first_lane + in.lanes > stride)
    return fail(BSB_INVALID_ARGUMENT, "first_lane + lanes exceeds the lanes of the row store");
  const uint32_t need = (1u << Q_EPISODE) | needed_quantities(kScoring[in.experiment].kind);
  ScoreSrc s;
  memset(&s, 0, sizeof(s));
  for (int q = 0; q < NUM_QUANTITIES; ++q) {
    const int32_t c = in.columns[q];
    if ((need >> q) & 1u) {
      if (c < 0 || c >= n_columns) return fail(BSB_INVALID_ARGUMENT, "a column the experiment's score needs is missing");
      s.col[q] = (int8_t)c;
    } else {
      s.col[q] = 0;
    }
  }
  s.rows = rows + in.first_lane; s.counts = counts + in.first_lane;
  s.stride = stride; s.key = in.group_key; s.ncols = (int32_t)n_columns; s.n_points = (int16_t)n_points;
  out->src = s; out->experiment = in.experiment; out->setting = in.setting; out->device = device;
  return BSB_OK;
}

}  // namespace

extern "C" int32_t bsb_score(const bsb_score_source* sources, int32_t count, int64_t lanes, double* scores,
                             uint8_t* finished, double* tag_scores, void* stream) {
  if (!sources || !scores || !finished || !tag_scores) return fail(BSB_INVALID_ARGUMENT, "null argument");
  if (count < 1 || count > BSB_SCORE_MAX_SOURCES)
    return fail(BSB_INVALID_ARGUMENT, "count must be in [1, BSB_SCORE_MAX_SOURCES]");
  if (lanes < 0) return fail(BSB_INVALID_ARGUMENT, "lanes must be >= 0");
  std::vector<Resolved> all((size_t)count);
  for (int32_t k = 0; k < count; ++k) {
    int rc = resolve(sources[k], lanes, &all[k]);
    if (rc != BSB_OK) return rc;
    if (all[k].device != all[0].device) return fail(BSB_INVALID_ARGUMENT, "sources live on different devices");
  }
  // Sorted by (experiment, group key, setting): each group is a run of sources in pandas' groupby order.
  std::sort(all.begin(), all.end(), [](const Resolved& a, const Resolved& b) {
    if (a.experiment != b.experiment) return a.experiment < b.experiment;
    if (a.src.key != b.src.key) return a.src.key < b.src.key;
    return a.setting < b.setting;
  });
  for (int32_t k = 1; k < count; ++k)
    if (all[k].experiment == all[k - 1].experiment && all[k].setting == all[k - 1].setting)
      return fail(BSB_INVALID_ARGUMENT, "the same setting is given twice");
  static ScoreJob job;       // host staging of the launch parameters (too large for the stack)
  static std::mutex job_lock;
  std::lock_guard<std::mutex> guard(job_lock);
  job.lanes = lanes;
  for (int e = 0; e < NUM_EXPERIMENTS; ++e) job.x[e] = kScoring[e];
  int32_t k = 0;
  for (int e = 0; e <= NUM_EXPERIMENTS; ++e) {
    while (k < count && all[k].experiment < e) ++k;
    job.begin[e] = k;
  }
  for (int32_t s = 0; s < count; ++s) job.src[s] = all[s].src;
  if (lanes == 0) return BSB_OK;
  const int device = all[0].device;
  if (device >= 0) {
    DeviceScope scope(device);
    const unsigned blocks = (unsigned)((lanes + kScoreThreads - 1) / kScoreThreads);
    cudaStream_t s = static_cast<cudaStream_t>(stream);
    score_kernel<<<dim3(blocks, NUM_EXPERIMENTS), kScoreThreads, 0, s>>>(job, scores, finished);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    BSB_CUDA(cudaGetLastError());
    score_tags_kernel<<<blocks, kScoreThreads, 0, s>>>(job, scores, tag_scores);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    BSB_CUDA(cudaGetLastError());
    return BSB_OK;
  }
  for (int e = 0; e < NUM_EXPERIMENTS; ++e)
    for (int64_t j = 0; j < lanes; ++j) {
      bool f;
      score_experiment(job.src + job.begin[e], job.begin[e + 1] - job.begin[e], job.x[e], j,
                       &scores[(int64_t)e * lanes + j], &f);
      finished[(int64_t)e * lanes + j] = f ? 1 : 0;
    }
  for (int64_t j = 0; j < lanes; ++j) tag_means(job, scores, j, tag_scores);
  return BSB_OK;
}
