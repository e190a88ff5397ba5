// bsuite scores from the per-lane log rows, written once as __host__ __device__ functions: the scoring kernel
// (bsb_score.cu) and the host path both call them.
//
// Each function restates one scoring rule of the reference's analysis code and cites it.  The reference scores a
// pandas DataFrame holding the CSV rows of one results directory (`summary_analysis.bsuite_score`); here one lane j
// plays that directory, and the rows of setting s are row k = 0 .. count-1 of source s at lane j.  Rows are recorded
// at strictly ascending episode counts no larger than the experiment's NUM_EPISODES (the Logging wrapper's schedule,
// utils/wrappers.py:140-147), which the rules below rely on:
//   - a setting's largest episode is its last row, so `df.episode == n_eps` with n_eps the largest episode of a
//     group selects at most the last row of each setting, and only those settings whose last row is at n_eps;
//   - the `episode <= NUM_EPISODES` filters (cartpole, cartpole_swingup, deep_sea) keep every row;
//   - the running maxima the reference takes over a column that only grows (best_episode: environments/cartpole.py:150,
//     experiments/cartpole_swingup/cartpole_swingup.py:119) are the last row's value.
// A score then reads O(1) rows per (lane, setting); deep_sea's first-solved scan and mnist's tail are the exceptions.
//
// Means follow numpy's pairwise summation (numpy/_core/src/umath/loops_utils.h.src, pairwise_sum) for up to 128
// values: a plain left-to-right sum below 8, otherwise 8 strided partial sums combined as
// ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)) and the remainder added in order.  pandas' Series.mean is that sum over the
// values with NaN replaced by 0, divided by the count of the others (pandas/core/nanops.py, nanmean).
#pragma once
#include <math.h>
#include <stdint.h>

#include "bsb_rng.cuh"   // BSB_HD

namespace bsb {

// Quantities a score reads (enum bsb_score_quantity): their column in a source's rows.
enum { Q_EPISODE = 0, Q_TOTAL_RETURN, Q_TOTAL_REGRET, Q_RAW_RETURN, Q_BEST_EPISODE, Q_TOTAL_PERFECT,
       Q_TOTAL_BAD_EPISODES, NUM_QUANTITIES };

// How an experiment is scored.
enum ScoreKind {
  SK_REGRET = 0,       // utils/plotting.py:57-65 ave_regret_score on total_regret (bandit, catch)
  SK_MNIST,            // mnist/analysis.py:31-42: regret + final accuracy
  SK_CARTPOLE,         // cartpole/analysis.py:32-50: regret on 1000 * episode - raw_return + a good run
  SK_MOUNTAIN_CAR,     // mountain_car/analysis.py:31-44: regret on -100 * episode - raw_return
  SK_SWINGUP,          // cartpole_swingup/analysis.py:32-54: per height_threshold, regret + a swing-up
  SK_DEEP_SEA,         // deep_sea/analysis.py:37-91 (find_solution, score)
  SK_DISCOUNTING,      // discounting_chain/analysis.py:33-38
  SK_MEMORY,           // memory_len/analysis.py:31-51
  SK_UMBRELLA,         // umbrella_length/analysis.py:32-40 (score_by_group)
};

enum { NUM_EXPERIMENTS = 23, NUM_TAGS = 7 };
// Tags in sorted order (the rows of tag_scores): summary_analysis.py:98-100 ALL_TAGS, sorted.
enum { T_BASIC = 1, T_CREDIT = 2, T_EXPLORATION = 4, T_GENERALIZATION = 8, T_MEMORY = 16, T_NOISE = 32, T_SCALE = 64 };

// The scoring constants of one experiment (bsb_score.cu holds the table, one cited entry per experiment).
struct ExperimentScoring {
  int32_t kind;
  int32_t scaled;          // 1: plotting.score_by_scaling over the group key (noise_scale / reward_scale)
  int32_t num_episodes;    // <experiment>/sweep.py NUM_EPISODES
  int32_t tags;            // T_* mask of <experiment>/sweep.py TAGS
  double base;             // BASE_REGRET of the regret kinds
  double thresh;           // deep_sea: the avg_bad_episodes threshold
  double min_episode;      // deep_sea_stochastic: rows before this episode are dropped
};

// The quantities each kind reads (beyond the episode column every kind reads).
BSB_HD uint32_t needed_quantities(int kind) {
  switch (kind) {
    case SK_REGRET: case SK_MNIST: case SK_UMBRELLA: return 1u << Q_TOTAL_REGRET;
    case SK_CARTPOLE: return (1u << Q_RAW_RETURN) | (1u << Q_BEST_EPISODE);
    case SK_MOUNTAIN_CAR: return 1u << Q_RAW_RETURN;
    case SK_SWINGUP: return (1u << Q_TOTAL_RETURN) | (1u << Q_BEST_EPISODE);
    case SK_DEEP_SEA: return 1u << Q_TOTAL_BAD_EPISODES;
    case SK_DISCOUNTING: return 1u << Q_TOTAL_RETURN;
    case SK_MEMORY: return 1u << Q_TOTAL_PERFECT;
  }
  return 0u;
}

// One setting's rows as the scorer sees them (48 bytes: the kernel takes up to kScoreMaxSources of them by value).
struct ScoreSrc {
  const double* rows;      // [n_points][ncols][stride], already advanced to the source's first lane
  const int32_t* counts;   // [stride], likewise
  int64_t stride;
  double key;              // the setting's group key (sweep value), sources are sorted by it within an experiment
  int32_t ncols;
  int16_t n_points;
  int8_t col[NUM_QUANTITIES];
};

// Lane j of the sources [begin, end) of one experiment.
struct LaneRows {
  const ScoreSrc* src;
  int64_t j;
  BSB_HD int count(int s) const {
    const int c = src[s].counts[j];
    return c < 0 ? 0 : (c > src[s].n_points ? src[s].n_points : c);
  }
  BSB_HD double at(int s, int k, int q) const {
    const ScoreSrc& r = src[s];
    return r.rows[((int64_t)k * r.ncols + r.col[q]) * r.stride + j];
  }
};

BSB_HD double score_nan() { return (double)NAN; }

// np.clip(x, 0, 1), NaN stays NaN.
BSB_HD double clip01(double x) { return x < 0.0 ? 0.0 : (x > 1.0 ? 1.0 : x); }

// numpy's pairwise sum of a stream of up to 128 values (see the file comment).
struct PairwiseSum {
  double r[8], b[8];
  int n;
  BSB_HD PairwiseSum() : n(0) {}
  BSB_HD void add(double x) {
    const int k = n & 7;
    b[k] = x;
    ++n;
    if (k == 7) {
      if (n == 8) { for (int i = 0; i < 8; ++i) r[i] = b[i]; }
      else { for (int i = 0; i < 8; ++i) r[i] += b[i]; }
    }
  }
  BSB_HD double sum() const {
    double s = 0.0;
    if (n >= 8) s = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
    for (int i = 0; i < (n & 7); ++i) s += b[i];
    return s;
  }
  BSB_HD double mean() const { return n ? sum() / (double)n : score_nan(); }
};

// pandas Series.mean: NaN counts as 0 in the sum and not in the count.
struct SkipNaNMean {
  PairwiseSum s;
  int valid;
  BSB_HD SkipNaNMean() : valid(0) {}
  BSB_HD void add(double x) { if (x == x) { s.add(x); ++valid; } else s.add(0.0); }
  BSB_HD double mean() const { return valid ? s.sum() / (double)valid : score_nan(); }
};

// The regret a row carries, per kind (the preprocess functions).
BSB_HD double row_regret(const LaneRows& L, int s, int k, int kind) {
  const double episode = L.at(s, k, Q_EPISODE);
  switch (kind) {
    case SK_CARTPOLE: return 1000.0 * episode - L.at(s, k, Q_RAW_RETURN);          // cartpole/analysis.py:45-50
    case SK_MOUNTAIN_CAR: return -100.0 * episode - L.at(s, k, Q_RAW_RETURN);      // mountain_car/analysis.py:38-44
    case SK_SWINGUP: return 700.0 * episode - L.at(s, k, Q_TOTAL_RETURN);          // cartpole_swingup/analysis.py:32-37
    case SK_MEMORY:                                                                 // memory_len/analysis.py:31-39
      return (episode - L.at(s, k, Q_TOTAL_PERFECT)) / 0.5;
  }
  return L.at(s, k, Q_TOTAL_REGRET);
}

// The largest episode of the sources [a, b) (their last rows), or -1 when they hold no row.
BSB_HD double max_episode(const LaneRows& L, int a, int b) {
  double m = -1.0;
  for (int s = a; s < b; ++s) {
    const int c = L.count(s);
    if (c > 0) { const double e = L.at(s, c - 1, Q_EPISODE); if (e > m) m = e; }
  }
  return m;
}

// mean(regret at n_eps) / n_eps over the sources [a, b): plotting.ave_regret_score's mean_regret
// (utils/plotting.py:57-65), memory_len's ave_perfection, umbrella's ave_regret, discounting_chain's ave_return.
BSB_HD double mean_at_last_episode(const LaneRows& L, int a, int b, int kind, double n_eps) {
  PairwiseSum m;
  for (int s = a; s < b; ++s) {
    const int c = L.count(s);
    if (c > 0 && L.at(s, c - 1, Q_EPISODE) == n_eps)
      m.add(kind == SK_DISCOUNTING ? L.at(s, c - 1, Q_TOTAL_RETURN) : row_regret(L, s, c - 1, kind));
  }
  return m.mean() / n_eps;
}

// plotting.ave_regret_score (utils/plotting.py:57-65): clip((base - mean_regret) / base, 0, 1).
BSB_HD double ave_regret_score(const LaneRows& L, int a, int b, int kind, double base, int num_episodes) {
  const double n_eps = fmin(max_episode(L, a, b), (double)num_episodes);
  return clip01((base - mean_at_last_episode(L, a, b, kind, n_eps)) / base);
}

// Fraction of the sources [a, b) with rows whose largest best_episode beats `good`
// (np.mean(df.groupby('bsuite_id')['best_episode'].max() > GOOD_EPISODE)).
BSB_HD double good_run_fraction(const LaneRows& L, int a, int b, double good) {
  int n = 0, hit = 0;
  for (int s = a; s < b; ++s) {
    const int c = L.count(s);
    if (c > 0) { ++n; hit += L.at(s, c - 1, Q_BEST_EPISODE) > good ? 1 : 0; }
  }
  return (double)hit / (double)n;
}

// mnist/analysis.py:36-41: 0.5 * mean(ave_return + 1) over the rows past 0.9 * NUM_EPISODES, where
// ave_return = 1 - diff(total_regret) / diff(episode) between consecutive rows of a setting; NaN without such rows.
BSB_HD double mnist_accuracy(const LaneRows& L, int a, int b, int num_episodes) {
  const double tail = 0.9 * (double)num_episodes;
  PairwiseSum m;
  for (int s = a; s < b; ++s) {
    const int c = L.count(s);
    int k = c;
    while (k > 0 && L.at(s, k - 1, Q_EPISODE) > tail) --k;
    for (k = k < 1 ? 1 : k; k < c; ++k) {
      const double d_regret = L.at(s, k, Q_TOTAL_REGRET) - L.at(s, k - 1, Q_TOTAL_REGRET);
      const double d_episode = L.at(s, k, Q_EPISODE) - L.at(s, k - 1, Q_EPISODE);
      m.add((1.0 - d_regret / d_episode) + 1.0);
    }
  }
  return m.mean() * 0.5;
}

// The score an experiment's score function gives the sources [a, b) (all of them, or one scaling group).
BSB_HD double base_score(const LaneRows& L, int a, int b, const ExperimentScoring& x) {
  switch (x.kind) {
    case SK_MNIST:
      return 0.5 * (ave_regret_score(L, a, b, x.kind, x.base, x.num_episodes) +
                    mnist_accuracy(L, a, b, x.num_episodes));
    case SK_CARTPOLE:
      return 0.5 * (ave_regret_score(L, a, b, x.kind, x.base, x.num_episodes) + good_run_fraction(L, a, b, 500.0));
    case SK_DISCOUNTING: {
      const double n_eps = fmin(max_episode(L, a, b), (double)x.num_episodes);
      return clip01(1.0 - 10.0 * (1.1 - mean_at_last_episode(L, a, b, x.kind, n_eps)));
    }
  }
  return ave_regret_score(L, a, b, x.kind, x.base, x.num_episodes);
}

// deep_sea/analysis.py:37-91 for one `size` group, sources [a, b): rows past the stochastic variant's first
// episodes (deep_sea_stochastic/analysis.py:42-58); the first episode with total_bad_episodes / episode < thresh,
// else the group is unsolved at its largest episode; 1 when solved before 2**size + 100 episodes.
// Returns -1 when the filter leaves the group no row.
BSB_HD int deep_sea_beats(const LaneRows& L, int a, int b, const ExperimentScoring& x) {
  double first = -1.0, last = -1.0;
  for (int s = a; s < b; ++s) {
    const int c = L.count(s);
    if (c == 0) continue;
    const double last_here = L.at(s, c - 1, Q_EPISODE);
    if (last_here < x.min_episode) continue;          // episodes ascend: the filter leaves this setting no row
    if (last_here > last) last = last_here;
    for (int k = 0; k < c; ++k) {
      const double episode = L.at(s, k, Q_EPISODE);
      if (episode < x.min_episode) continue;
      if (L.at(s, k, Q_TOTAL_BAD_EPISODES) / episode < x.thresh) {
        if (first < 0.0 || episode < first) first = episode;
        break;
      }
    }
  }
  if (last < 0.0) return -1;
  return first >= 0.0 && first < ldexp(1.0, (int)L.src[a].key) + 100.0 ? 1 : 0;
}

// Does experiment e hold a row at lane j?
BSB_HD bool experiment_present(const ScoreSrc* src, int n, int64_t j) {
  const LaneRows L{src, j};
  for (int s = 0; s < n; ++s) if (L.count(s) > 0) return true;
  return false;
}

// Score of an experiment at lane j from its sources [0, n) (sorted by group key), and whether every setting that
// has rows reached NUM_EPISODES (summary_analysis.py:103-108, _is_finished).  An experiment without rows scores NaN, unfinished.
BSB_HD void score_experiment(const ScoreSrc* src, int n, const ExperimentScoring& x, int64_t j, double* score,
                             bool* finished) {
  const LaneRows L{src, j};
  bool any = false, done = true;
  for (int s = 0; s < n; ++s) {
    const int c = L.count(s);
    if (c > 0) { any = true; done = done && L.at(s, c - 1, Q_EPISODE) >= (double)x.num_episodes; }
  }
  *finished = any && done;
  if (!any) { *score = score_nan(); return; }
  // Groups: runs of equal keys, each with at least one row (pandas' groupby sees only rows).
  if (x.kind == SK_SWINGUP || x.kind == SK_MEMORY || x.kind == SK_UMBRELLA || x.kind == SK_DEEP_SEA || x.scaled) {
    PairwiseSum group_scores;
    double kept[8];     // score_by_scaling's per-group scores (5 noise / reward scales in the sweep)
    int n_kept = 0;
    for (int a = 0; a < n;) {
      int b = a + 1;
      while (b < n && src[b].key == src[a].key) ++b;
      if (max_episode(L, a, b) >= 0.0) {
        double g;
        if (x.kind == SK_DEEP_SEA) {
          const int beats = deep_sea_beats(L, a, b, x);
          if (beats < 0) { a = b; continue; }
          g = (double)beats;
        } else if (x.kind == SK_SWINGUP) {
          g = 0.5 * (ave_regret_score(L, a, b, x.kind, x.base, x.num_episodes) + good_run_fraction(L, a, b, 100.0));
        } else if (x.kind == SK_MEMORY || x.kind == SK_UMBRELLA) {
          const double n_eps = fmin(max_episode(L, a, b), (double)x.num_episodes);
          g = mean_at_last_episode(L, a, b, x.kind, n_eps) < x.thresh ? 1.0 : 0.0;
        } else {
          g = base_score(L, a, b, x);
          if (n_kept < 8) kept[n_kept] = g;
          ++n_kept;
        }
        group_scores.add(g);
      }
      a = b;
    }
    if (!x.scaled) { *score = group_scores.mean(); return; }
    // plotting.score_by_scaling (utils/plotting.py:68-77): 0.5 * (clip(mean) + clip(mean - std)), np.std ddof 0
    const double mean = group_scores.mean();
    PairwiseSum sq;
    for (int g = 0; g < n_kept && g < 8; ++g) sq.add((kept[g] - mean) * (kept[g] - mean));
    const double std_dev = sqrt(sq.sum() / (double)n_kept);
    *score = 0.5 * (clip01(mean) + clip01(mean - std_dev));
    return;
  }
  *score = base_score(L, 0, n, x);
}

}  // namespace bsb
