// Host path and kernel launch, instantiated once per kernel variant in the translation unit the variant list gives it
// (bsb_variants.cu).
#pragma once
#include <cstring>
#include <type_traits>
#include <vector>

#include "bsb_env.h"

namespace bsb {

// --------------------------- host path --------------------------------------
template <class F> struct HostEmit {
  template <class R> static void run(const EnvParams& p, const typename F::Lane& L, R&, float* dst) { F::row(p, L, dst, 1); }
};
template <> struct HostEmit<UmbrellaChain> {
  template <class R> static void run(const EnvParams& p, const UmbrellaChain::Lane& L, R& r, float* dst) { UmbrellaChain::row(p, L, r, dst, 1); }
};
template <> struct HostEmit<DeepSea> {
  template <class R> static void run(const EnvParams& p, const DeepSea::Lane& L, R&, float* dst) {
    for (int e = 0; e < p.obs_numel; ++e) dst[e] = 0.f;
    if (L.hot >= 0) dst[L.hot] = 1.f;
  }
};
template <> struct HostEmit<Catch> {
  template <class R> static void run(const EnvParams& p, const Catch::Lane& L, R&, float* dst) {
    for (int e = 0; e < p.obs_numel; ++e) dst[e] = 0.f;
    dst[L.hot_a] = 1.f; dst[L.hot_b] = 1.f;
  }
};
template <> struct HostEmit<Mnist> {
  template <class R> static void run(const EnvParams& p, const Mnist::Lane& L, R&, float* dst) {
    if (L.image < 0) { for (int e = 0; e < p.obs_numel; ++e) dst[e] = 0.f; return; }
    const int8_t* src = p.images + (int64_t)L.image * p.obs_numel;
    for (int e = 0; e < p.obs_numel; ++e) dst[e] = Mnist::pixel(src[e]);
  }
};

// Observations of type O other than float32: each lane's float32 observation is rendered into `f32` and converted
// element by element with obs_cast, the function the kernels use.  kSameStep: a lane whose step returned LAST is reset
// in the same call, and its final observation goes to a.final_obs when that is given.  kPacked: every lane runs with
// its setting's parameters (pack_lane_params), as the packed kernels do.  kRagged: the same with ragged_setting_params,
// and lane j of setting k writes row j of the setting's observation block.  `mask` (masked calls and rollouts): lane i
// acts only while mask[i] != 0 and its budget episodes_left[i] (when given) is positive; each LAST it returns takes one
// from the budget, so its active steps are a prefix of the T.  The calls it sits out come after them
// (lane_sit_out_calls), and their outputs are not written.  No observation buffer (bsb_advance_masked): nothing is
// rendered, and each observation's random draws are made without it (ObsDraws::skip), as the kernel does.
template <class V, int RK>
void host_run(const EnvParams& p, const LaunchArgs& a, const uint8_t* mask = nullptr, int64_t* episodes_left = nullptr) {
  typedef typename V::Fam F;
  typedef typename V::Obs O;
  constexpr bool kSameStep = V::kSameStep, kPacked = V::kPacked, kRagged = V::kRagged;
  typedef typename RngOf<RK>::type R;
  const int64_t B = p.batch;
  const int K = p.obs_numel;
  O* const obs = reinterpret_cast<O*>(a.obs);
  const RaggedTable* ragged = kRagged ? reinterpret_cast<const RaggedTable*>(p.pack) : nullptr;
  O* const fin = reinterpret_cast<O*>(a.final_obs);
  std::vector<float> f32(std::is_same<O, float>::value ? 0 : (size_t)K);
  const bool noise = p.wrapper == BSB_WRAP_REWARD_NOISE && a.mode != MODE_INIT;
  const bool track = p.ep != nullptr && a.mode != MODE_INIT;
  const MailFields out = {a.reward, a.reward_f64, a.discount, a.step_type};
  EnvParams setting_p;                    // packed handles: p with the current lane's setting
  auto render = [&](const EnvParams& lp, const typename F::Lane& L, R& rng, O* dst) {
    if constexpr (std::is_same<O, float>::value) {
      HostEmit<F>::run(lp, L, rng, dst);
    } else {
      HostEmit<F>::run(lp, L, rng, f32.data());
      for (int e = 0; e < K; ++e) dst[e] = obs_cast<O>(f32[(size_t)e]);
    }
  };
  for (int64_t lane = 0; lane < B; ++lane) {
    const bool budgeted = mask && mask[lane] && episodes_left;
    int64_t left = budgeted ? episodes_left[lane] : 0;
    if ((mask && !mask[lane]) || (budgeted && left <= 0)) {
      if (track) lane_sit_out_calls(p, lane, a.T);
      continue;
    }
    if constexpr (kPacked) { setting_p = p; pack_lane_params(setting_p, lane); }
    O* lane_obs = obs ? obs + lane * (int64_t)K : nullptr;      // step 0's observation row of this lane
    int64_t step_elems = B * (int64_t)K;
    if constexpr (kRagged) {
      const int64_t k = lane / ragged->pack.lanes_per_setting;
      const RaggedSetting& s = ragged_setting(ragged, k);
      setting_p = p;
      ragged_setting_params(setting_p, s, ragged->mapping_bits);
      if (obs) lane_obs = obs + s.obs_offset + (lane - s.lane_shift) * (int64_t)s.obs_numel;
      step_elems = ragged->step_elems;
    }
    const EnvParams& lp = (kPacked || kRagged) ? setting_p : p;
    typename F::Lane L;
    R rng, wrng;
    EpisodeStats ep;
    ActionStream action_stream;
    action_stream.open();
    lane_open<F>(lp, lane, L, rng, wrng, ep, a.mode, noise, track);
    if (a.mode == MODE_INIT) F::ctor_draws(lp, L, rng);
    MergedReset<F, R> merged;
    F::init(p, merged.last);
    merged.done = false;
    int64_t acted = 0;
    for (int64_t t = 0; t < a.T; ++t) {
      const int64_t off = t * B + lane;
      int32_t action = 0;
      if (a.mode == MODE_STEP) {
        action = a.actions ? a.actions[off]
                           : action_stream.sample(a.action_seed, lp.lane_offset + (uint64_t)lane, (uint64_t)(a.step0 + t), p.num_actions);
        if (a.actions_out) a.actions_out[off] = action;
      }
      lane_step<F, R, kSameStep>(lp, lane, L, rng, wrng, ep, action, a.mode, noise, track, a.step0 + t, out, off, &merged);
      if constexpr (kSameStep) { if (merged.done && fin) render(lp, merged.last, merged.rng, fin + off * (int64_t)K); }
      if (obs) render(lp, L, rng, lane_obs + t * step_elems);
      else ObsDraws<F>::skip(lp, rng);      // bsb_advance_masked: the observation's draws, not the observation
      ++acted;
      // the step's LAST: a same-step lane's merged reset, else the _reset_next_step flag the step left set
      if (budgeted && (kSameStep ? merged.done : L.nr != 0) && --left == 0) break;
    }
    lane_close<F>(lp, lane, L, rng, wrng, ep, noise, track);
    if (mask && track && acted < a.T) lane_sit_out_calls(p, lane, a.T - acted);
    if (budgeted) episodes_left[lane] = left;
  }
}

// --------------------------- device dispatch --------------------------------
// Launch geometry, shared by the launchers of both kernels.
struct Geometry { int threads = 0; size_t smem = 0; int64_t n_chunks = 0, grid = 0; int extra_blocks = 0; };

// The chunks of `cl` lanes a launch deals: a ragged pack's setting k owns ceil(L / cl) of them, so no chunk straddles
// two settings; every other handle is one block of B lanes.
inline int64_t launch_chunks(const bsb_env* e, bool ragged, int cl) {
  const int64_t lanes = ragged ? e->lanes_per_setting : e->p.batch;
  return (ragged ? (int64_t)e->n_settings : 1) * ((lanes + cl - 1) / cl);
}

// Chunk lanes, emitter plan (group lanes, stage rows), CTA size, shared memory and grid of a launch; fills a's
// emitter fields and, for a persistent grid (the deep_sea and mnist bulk paths, once the grid exceeds what is
// resident), its chunk counter.  `extra_threads` > 0 (the copiers of two-phase host steps) puts g.extra_blocks
// blocks of that many threads in all (at least one) in front of the chunk owners.
// kRagged (float32 observations, the settings' shapes in e->obs_rows / obs_cols, their deep_sea group sizes in
// e->group_lanes): the same rules with the chunks of ragged_chunks.  Row stages are sized for the largest K.  deep_sea
// tiles keep the grouped bulk store and its persistent grid, each setting with its own group size; the stage holds two
// of the largest group (a.group_lanes * p.obs_numel elements each, p.obs_numel being the largest K).  On compressible
// memory, where a batch of the same size would turn to compare-then-store or streaming stores, every chunk uses the
// streaming stores.
template <class F, class O, bool kRagged = false>
int plan_launch(bsb_env* e, LaunchArgs& a, Geometry& g, int extra_threads = 0) {
  const int K = e->p.obs_numel;
  const bool is_onehot = EmitKind<F>::value == EMIT_ONEHOT;
  const bool is_image = EmitKind<F>::value == EMIT_IMAGE;
  const int64_t B = e->p.batch;
  a.emit_bulk = 1;
  a.group_lanes = 1;
  a.work_counter = nullptr;
  a.work_base = 0;
  // Row / board stages per warp: two (the next row block is rendered while the TMA unit still reads the previous
  // one) unless that costs resident warps -- 16 warps per SM fit the register budget, so a warp can afford
  // ~14 KB of shared memory.  umbrella_distract (103-float rows, 13 KB per stage) would hold 8 warps per SM
  // with two stages and is bound by integer-multiply latency, not by the store.
  const size_t elem = sizeof(O);                     // bytes per observation element (obs_dtype)
  a.stage_rows = ((size_t)2 * 32 * (size_t)K * elem <= 14 * 1024) ? 2 : 1;
  // A single-step launch gives every warp exactly one row block to emit: the second stage would only be zeroed
  // (catch) and hold shared memory that another CTA could use.
  if (a.T == 1 && (EmitKind<F>::value == EMIT_ROWS || EmitKind<F>::value == EMIT_TWOHOT)) a.stage_rows = 1;
  a.cta_extra_elems = 0;
  a.bad_action = e->bad_action_dev;
  // Lanes per chunk.  The image emitter walks the chunk's lanes a few 3 KB tiles at a time, so it is bound by how
  // many warps share the batch: keep >= 4 warps per SM by halving the chunk (down to 8 lanes) when 32-lane chunks
  // would not.  The deep_sea bulk path keeps 32 (fewer, larger TMA stores win there).
  int chunk = 32;
  if (is_image)
    while (chunk > 8 && (B + chunk - 1) / chunk < 4 * (int64_t)e->num_sms) chunk >>= 1;
  a.chunk_lanes = chunk;
  g.n_chunks = launch_chunks(e, kRagged, chunk);
  int threads = 64;         // one chunk per warp: small CTAs spread evenly over the SMs (transition_kernel)
  bool persistent = false;
  const size_t tile = (size_t)K * elem;
  // deep_sea tiles written to compressible memory (bsb_obs_malloc) once the batch fills the GPU (>= 4 chunks per SM)
  // skip the bulk path, which gains nothing from compression there.  A launch of one step compares every tile with
  // what the destination holds and stores only the lines that differ (emit_onehot_reuse): compressed one-hot tiles
  // read back faster than any emitter can write them.  Fused rollouts (T > 1) ran slower that way and keep the 16-byte
  // streaming stores.  Smaller batches keep the bulk path, which overlaps a warp's stores with its next steps
  // (DESIGN.md §7, "Compressible observation memory").
  a.emit_reuse = 0;
  if (is_onehot && a.emit_bulk && g.n_chunks >= 4 * (int64_t)e->num_sms && in_compressed_block(a.obs)) {
    a.emit_bulk = 0;
    a.emit_reuse = a.T == 1 && !kRagged ? 1 : 0;
  }
  if (is_onehot && a.emit_bulk) {
    int m;                                  // lanes per bulk store
    if constexpr (kRagged) {
      int64_t largest = 0;
      for (int32_t k = 0; k < e->n_settings; ++k) {
        const int64_t elems = (int64_t)e->group_lanes[k] * e->obs_rows[k] * e->obs_cols[k];
        largest = elems > largest ? elems : largest;
      }
      m = (int)((largest + K - 1) / K);
    } else {
      m = tile_group_lanes(tile);
    }
    if (m == 0) {
      a.emit_bulk = 0;                      // tiles too large (or misaligned) for the staged path: vector stores
    } else {
      a.group_lanes = m; threads = 32; persistent = true;
    }
  }
  if (is_image && a.emit_bulk) {
    // mnist through the TMA unit: groups of m tiles staged in shared memory + mz all-zero tiles per CTA for the LAST
    // frames.  16-byte image loads need K % 16 == 0 (28 x 28 = 784 is).  ONE staging buffer of m <= 4 tiles per warp
    // and mz <= 8 zero tiles per CTA, each halved until it fits 28 KB.  28 x 28 in float32: m = 4 (12.25 KB, plus
    // the 1 KB pixel table: 13.25 KB per warp) and mz = 8 (24.5 KB, shared by the CTA's warps): 77.5 KB per
    // 128-thread CTA -> 2 CTAs = 8 warps per SM (64-thread CTAs: 51 KB -> 4 CTAs, also 8 warps).  The pixel
    // conversion is issue-bound, so resident warps matter more than overlapping a warp's own fill with its own store
    // (other warps fill that gap); the zero frames, pure bandwidth, leave in 24.5 KB stores.
    int m = 4;
    while (m > 1 && (size_t)m * tile > 28 * 1024) m >>= 1;
    int mz = 8;
    while (mz > 1 && (size_t)mz * tile > 28 * 1024) mz >>= 1;
    if ((K & 15) != 0 || (size_t)m * tile > 64 * 1024) {
      a.emit_bulk = 0;
    } else {
      a.group_lanes = m; a.stage_rows = 1; threads = 128; a.cta_extra_elems = mz * K; persistent = true;
      if (g.n_chunks < 2 * (int64_t)e->num_sms) threads = 64;      // small batches: more, smaller CTAs
    }
  }
  a.use_pdl = (a.mode == MODE_STEP && a.T == 1) ? 1 : 0;
  size_t per_warp = smem_elems_per_warp<F, O>(K, a.emit_bulk != 0, a.emit_reuse != 0, a.group_lanes, a.stage_rows) * elem;
  if ((EmitKind<F>::value == EMIT_ROWS || EmitKind<F>::value == EMIT_TWOHOT) && per_warp > 96 * 1024) {
    // rows / boards too long for a per-warp stage: long rows always get ONE stage (above), so the limit is
    // 32 * K * 4 bytes > 96 KB, i.e. K > 768 in float32 (catch boards of more than 768 cells such as 28 x 28,
    // umbrella_chain with more than 765 distractors), K > 1 536 in bfloat16, K > 3 072 in uint8: boards fall back to
    // shuffle-rendered vector stores, rows are rendered in place
    a.emit_bulk = 0; a.stage_rows = 0; per_warp = 0;
  }
  const size_t cta_extra = (size_t)a.cta_extra_elems * elem;
  size_t smem = per_warp * (size_t)(threads / 32) + cta_extra;
  while (smem > 96 * 1024 && threads > 32) { threads >>= 1; smem = per_warp * (size_t)(threads / 32) + cta_extra; }
  if (smem > 200 * 1024) return fail(BSB_UNSUPPORTED, "observation too large for the staged emitter");
  g.threads = threads;
  g.smem = smem;
  g.extra_blocks = extra_threads > 0 ? (extra_threads / threads > 1 ? extra_threads / threads : 1) : 0;
  g.grid = (g.n_chunks + threads / 32 - 1) / (threads / 32) + g.extra_blocks;
  if (persistent) {
    // As many CTAs as are co-resident (shared-memory bound; 1 KB per CTA is reserved by the driver); their warps
    // draw chunks from the environment's global counter.
    int64_t per_sm = (int64_t)((227 * 1024) / (smem + 1024));
    per_sm = per_sm < 1 ? 1 : (per_sm > 16 ? 16 : per_sm);
    const int64_t resident = (int64_t)e->num_sms * per_sm;
    if (g.grid > resident) {      // else everything is resident anyway: one chunk per warp
      g.grid = resident;
      a.work_counter = a.clock ? a.clock + CLOCK_CHUNK : e->work_counter;
      a.work_base = a.clock ? 0ull : e->work_base;
    }
  }
  return BSB_OK;
}

template <class Kernel, class... Args>
int launch(bsb_env* e, const LaunchArgs& a, const Geometry& g, cudaStream_t stream, Kernel kernel, const Args&... args) {
  if (g.smem > 48 * 1024) BSB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)g.smem));
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)g.grid);
  cfg.blockDim = dim3((unsigned)g.threads);
  cfg.dynamicSmemBytes = g.smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  if (a.use_pdl) {
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
  }
  BSB_CUDA(cudaLaunchKernelEx(&cfg, kernel, args...));
  // chunks [warps, n_chunks) are fetched once each and every warp makes exactly one failing fetch
  // (graph-safe mode: the last CTA zeroes the counter instead)
  if (a.work_counter && !a.clock) e->work_base += (unsigned long long)g.n_chunks + (unsigned long long)(g.extra_blocks * (g.threads / 32));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return BSB_OK;
}

// Two-phase host step (DeepSea, Catch): one launch per step.
template <class V, int RK, bool kNoise, bool kTrack>
int two_phase_launch(bsb_env* e, LaunchArgs a, TwoPhaseArgs h, cudaStream_t stream) {
  if (a.clock) return fail(BSB_INTERNAL, "a host step reached graph-safe mode, which turns the mailbox path off");
  // Copiers: enough of them for ~512 threads, i.e. ~64 KB of 16-byte loads in flight.
  Geometry g;
  const int rc = plan_launch<typename V::Fam, typename V::Obs>(e, a, g, 512);
  if (rc != BSB_OK) return rc;
  h.copiers = g.extra_blocks;
  return launch(e, a, g, stream, two_phase_host_kernel<V, RK, kNoise, kTrack>, e->p, a, h);
}

// Runs `launch(noise, track)` with the template flags of the launch's wrappers (none for the constructor).
template <class Launch>
int with_flags(const bsb_env* e, const LaunchArgs& a, Launch launch) {
  const bool noise = e->p.wrapper == BSB_WRAP_REWARD_NOISE && a.mode != MODE_INIT;
  const bool track = e->p.ep != nullptr && a.mode != MODE_INIT;
  if (noise) return track ? launch(std::true_type(), std::true_type()) : launch(std::true_type(), std::false_type());
  return track ? launch(std::false_type(), std::true_type()) : launch(std::false_type(), std::false_type());
}

// The host path of variant V with the handle's bit source (unmasked calls: no mask, no budgets).
template <class V>
void run_host(const bsb_env* e, const LaunchArgs& a, const uint8_t* mask = nullptr, int64_t* episodes_left = nullptr) {
  if constexpr (Compiled<V>::kMt) {
    if (e->p.rng_kind == BSB_RNG_MT19937) return host_run<V, 1>(e->p, a, mask, episodes_left);
  }
  host_run<V, 0>(e->p, a, mask, episodes_left);
}

// bsb_step_budgeted on a host handle, as masked_kernel's CALL_BUDGETED runs it: every masked-in lane's current
// entries of a's outputs go to `previous` (observation rows as raw bytes), then the masked step with budgets, then the
// mask is cleared for the masked-in lanes whose budget was spent before the call.
template <class V>
void host_budgeted(const bsb_env* e, const LaunchArgs& a, uint8_t* mask, int64_t* episodes_left,
                   const bsb_outputs* previous) {
  typedef typename V::Obs O;
  const EnvParams& p = e->p;
  const int64_t B = p.batch;
  const RaggedTable* ragged = V::kRagged ? reinterpret_cast<const RaggedTable*>(p.pack) : nullptr;
  const O* obs = reinterpret_cast<const O*>(a.obs);
  O* prev_obs = reinterpret_cast<O*>(previous->observation);
  const O* fin = reinterpret_cast<const O*>(a.final_obs);
  O* prev_fin = reinterpret_cast<O*>(previous->final_observation);
  std::vector<uint8_t> spent((size_t)B, 0);
  for (int64_t lane = 0; lane < B; ++lane) {
    if (!mask[lane]) continue;
    spent[(size_t)lane] = episodes_left[lane] <= 0;
    int64_t row = lane * (int64_t)p.obs_numel, K = p.obs_numel;
    if constexpr (V::kRagged) {
      const RaggedSetting& s = ragged_setting(ragged, lane / ragged->pack.lanes_per_setting);
      row = s.obs_offset + (lane - s.lane_shift) * (int64_t)s.obs_numel;
      K = s.obs_numel;
    }
    memcpy(prev_obs + row, obs + row, (size_t)K * sizeof(O));
    if (fin && prev_fin) memcpy(prev_fin + lane * (int64_t)p.obs_numel, fin + lane * (int64_t)p.obs_numel, (size_t)p.obs_numel * sizeof(O));
    if (a.reward && previous->reward) previous->reward[lane] = a.reward[lane];
    if (a.reward_f64 && previous->reward_f64) previous->reward_f64[lane] = a.reward_f64[lane];
    if (a.discount && previous->discount) previous->discount[lane] = a.discount[lane];
    if (a.step_type && previous->step_type) previous->step_type[lane] = a.step_type[lane];
  }
  run_host<V>(e, a, mask, episodes_left);
  for (int64_t lane = 0; lane < B; ++lane)
    if (spent[(size_t)lane]) mask[lane] = 0;
}

// bsb_step_budgeted_policy on a host handle, as masked_kernel's CALL_POLICY runs it: every masked-in lane with budget
// left picks its action from its row of the policy's values (select_action; an invalid row raises the invalid-action
// flag) and writes it to a.actions_out, then host_budgeted steps with those actions.  Rows of other lanes are not read.
template <class V>
void host_policy(const bsb_env* e, const LaunchArgs& a, uint8_t* mask, int64_t* episodes_left,
                 const bsb_outputs* previous, const bsb_policy& policy) {
  const EnvParams& p = e->p;
  const int64_t B = p.batch;
  const RaggedTable* ragged = V::kRagged ? reinterpret_cast<const RaggedTable*>(p.pack) : nullptr;
  std::vector<int32_t> actions((size_t)B, 0);
  for (int64_t lane = 0; lane < B; ++lane) {
    if (!mask[lane] || episodes_left[lane] <= 0) continue;
    EnvParams lp = p;                     // the lane's setting: its lane_offset keys the stream as the kernel's does
    if constexpr (V::kRagged) {
      ragged_setting_params(lp, ragged_setting(ragged, lane / ragged->pack.lanes_per_setting), ragged->mapping_bits);
    } else if constexpr (V::kPacked) {
      pack_lane_params(lp, lane);
    }
    bool invalid = false;
    const int32_t action = select_action(policy.kind, policy.values + lane * (int64_t)p.num_actions, p.num_actions,
                                         policy.epsilon, policy.seed, lp.lane_offset + (uint64_t)lane,
                                         (uint64_t)a.step0, invalid);
    if (invalid && e->bad_action_host) *e->bad_action_host = 1;
    actions[(size_t)lane] = action;
    if (a.actions_out) a.actions_out[lane] = action;
  }
  LaunchArgs chosen = a;
  chosen.actions = actions.data();
  chosen.actions_out = nullptr;
  host_budgeted<V>(e, chosen, mask, episodes_left, previous);
}

// The step of a recorded or sequence step on a host handle (CALL_RECORD's and CALL_SEQUENCE's): host_policy (a
// policy) or host_budgeted (the caller's actions).  `stepped[i]`: lane i stepped (mask set, budget left before the
// call); `used[i]`: the action it stepped with.
template <class V>
void host_step_used(const bsb_env* e, const LaunchArgs& a, uint8_t* mask, int64_t* episodes_left,
                    const bsb_outputs* previous, const bsb_policy* policy, std::vector<uint8_t>& stepped,
                    std::vector<int32_t>& used) {
  const EnvParams& p = e->p;
  const int64_t B = p.batch;
  stepped.assign((size_t)B, 0);
  used.assign((size_t)B, 0);
  for (int64_t lane = 0; lane < B; ++lane) {
    stepped[(size_t)lane] = mask[lane] && episodes_left[lane] > 0;
    if (stepped[(size_t)lane] && !policy) {
      const int32_t action = a.actions[lane];
      used[(size_t)lane] = (uint32_t)action < (uint32_t)p.num_actions ? action : (action < 0 ? 0 : p.num_actions - 1);
    }
  }
  if (policy) {
    LaunchArgs picked = a;
    picked.actions_out = used.data();
    host_policy<V>(e, picked, mask, episodes_left, previous, *policy);
    if (a.actions_out)
      for (int64_t lane = 0; lane < B; ++lane)
        if (stepped[(size_t)lane]) a.actions_out[lane] = used[(size_t)lane];
  } else {
    host_budgeted<V>(e, a, mask, episodes_left, previous);
  }
}

// bsb_step_budgeted_record on a host handle, as masked_kernel's CALL_RECORD runs it: host_step_used, then every lane
// that stepped and whose new step type is not FIRST appends its transition to slot num_added % capacity of its ring:
// o_tm1 from `previous`, o_t from the new observation row (a same-step LAST: the final observation row), as raw bytes.
template <class V>
void host_record(const bsb_env* e, const LaunchArgs& a, uint8_t* mask, int64_t* episodes_left,
                 const bsb_outputs* previous, const bsb_policy* policy, const bsb_replay& r) {
  typedef typename V::Obs O;
  const EnvParams& p = e->p;
  const int64_t B = p.batch;
  const RaggedTable* ragged = V::kRagged ? reinterpret_cast<const RaggedTable*>(p.pack) : nullptr;
  const int64_t step_elems = V::kRagged ? ragged->step_elems : B * (int64_t)p.obs_numel;
  std::vector<uint8_t> stepped;
  std::vector<int32_t> used;
  host_step_used<V>(e, a, mask, episodes_left, previous, policy, stepped, used);
  const O* prev_obs = reinterpret_cast<const O*>(previous->observation);
  const O* obs = reinterpret_cast<const O*>(a.obs);
  const O* fin = reinterpret_cast<const O*>(a.final_obs);
  O* ring_tm1 = reinterpret_cast<O*>(r.obs_tm1);
  O* ring_obs = reinterpret_cast<O*>(r.next.observation);
  for (int64_t lane = 0; lane < B; ++lane) {
    const int32_t type = a.step_type[lane];
    if (!stepped[(size_t)lane] || type == FIRST) continue;
    const int64_t n = r.num_added[lane];
    const int64_t slot = n % r.capacity;
    r.num_added[lane] = n + 1;
    const int64_t at = slot * B + lane;
    r.action[at] = used[(size_t)lane];
    if (r.next.reward) r.next.reward[at] = a.reward ? a.reward[lane] : (float)a.reward_f64[lane];
    if (r.next.reward_f64) r.next.reward_f64[at] = a.reward_f64 ? a.reward_f64[lane] : (double)a.reward[lane];
    if (r.next.discount) r.next.discount[at] = a.discount[lane];
    if (r.next.step_type) r.next.step_type[at] = type;
    int64_t row = lane * (int64_t)p.obs_numel, K = p.obs_numel;
    if constexpr (V::kRagged) {
      const RaggedSetting& s = ragged_setting(ragged, lane / ragged->pack.lanes_per_setting);
      row = s.obs_offset + (lane - s.lane_shift) * (int64_t)s.obs_numel;
      K = s.obs_numel;
    }
    const bool final_row = V::kSameStep && type == LAST;
    memcpy(ring_tm1 + slot * step_elems + row, prev_obs + row, (size_t)K * sizeof(O));
    memcpy(ring_obs + slot * step_elems + row, (final_row ? fin : obs) + row, (size_t)K * sizeof(O));
  }
}

// bsb_step_budgeted_sequence on a host handle, as masked_kernel's CALL_SEQUENCE runs it: host_step_used, then every
// lane that stepped and whose new step type is not FIRST appends its transition at entry t of its sequence (t = 0
// after a full sequence or a LAST, with o_tm1 from `previous` at observation slot 0), and every lane's ready flag is
// written.  Rows move as raw bytes.
template <class V>
void host_sequence(const bsb_env* e, const LaunchArgs& a, uint8_t* mask, int64_t* episodes_left,
                   const bsb_outputs* previous, const bsb_policy* policy, const bsb_sequence& q) {
  typedef typename V::Obs O;
  const EnvParams& p = e->p;
  const int64_t B = p.batch;
  const RaggedTable* ragged = V::kRagged ? reinterpret_cast<const RaggedTable*>(p.pack) : nullptr;
  const int64_t step_elems = V::kRagged ? ragged->step_elems : B * (int64_t)p.obs_numel;
  std::vector<uint8_t> stepped;
  std::vector<int32_t> used;
  host_step_used<V>(e, a, mask, episodes_left, previous, policy, stepped, used);
  const O* prev_obs = reinterpret_cast<const O*>(previous->observation);
  const O* obs = reinterpret_cast<const O*>(a.obs);
  const O* fin = reinterpret_cast<const O*>(a.final_obs);
  O* seq = reinterpret_cast<O*>(q.observations);
  const int64_t T = q.max_length;
  for (int64_t lane = 0; lane < B; ++lane) {
    const int32_t type = a.step_type[lane];
    if (!stepped[(size_t)lane] || type == FIRST) {
      q.ready[lane] = 0;
      continue;
    }
    int64_t t = q.length[lane];
    if ((uint64_t)t >= (uint64_t)T || (t > 0 && q.next.step_type[(t - 1) * B + lane] == LAST)) t = 0;
    const int64_t at = t * B + lane;
    q.action[at] = used[(size_t)lane];
    if (q.next.reward) q.next.reward[at] = a.reward ? a.reward[lane] : (float)a.reward_f64[lane];
    if (q.next.reward_f64) q.next.reward_f64[at] = a.reward_f64 ? a.reward_f64[lane] : (double)a.reward[lane];
    q.next.discount[at] = a.discount[lane];
    q.next.step_type[at] = type;
    q.length[lane] = t + 1;
    q.ready[lane] = t + 1 == T || type == LAST ? 1 : 0;
    int64_t row = lane * (int64_t)p.obs_numel, K = p.obs_numel;
    if constexpr (V::kRagged) {
      const RaggedSetting& s = ragged_setting(ragged, lane / ragged->pack.lanes_per_setting);
      row = s.obs_offset + (lane - s.lane_shift) * (int64_t)s.obs_numel;
      K = s.obs_numel;
    }
    const bool final_row = V::kSameStep && type == LAST;
    if (t == 0) memcpy(seq + row, prev_obs + row, (size_t)K * sizeof(O));
    memcpy(seq + (t + 1) * step_elems + row, (final_row ? fin : obs) + row, (size_t)K * sizeof(O));
  }
}

// bsb_step_budgeted_ensemble on a host handle, as masked_kernel's CALL_ENSEMBLE runs it: every lane that steps (mask
// set, budget left) reads head h = heads[lane] (clamped into [0, K), raising the invalid-action flag, when outside it)
// and its row (h, lane) of the values is gathered into a [B, A] policy; host_record (a replay) or host_policy steps
// with it; then every such lane whose step ended an episode -- its budget counted down -- draws its new head.
template <class V>
void host_ensemble(const bsb_env* e, const LaunchArgs& a, uint8_t* mask, int64_t* episodes_left,
                   const bsb_outputs* previous, const bsb_policy& policy, const bsb_ensemble_policy& ens,
                   const bsb_replay* replay) {
  const EnvParams& p = e->p;
  const int64_t B = p.batch, A = p.num_actions;
  const RaggedTable* ragged = V::kRagged ? reinterpret_cast<const RaggedTable*>(p.pack) : nullptr;
  std::vector<float> rows((size_t)(B * A), 0.f);
  std::vector<int64_t> before(episodes_left, episodes_left + B);
  std::vector<uint8_t> stepped((size_t)B, 0);
  for (int64_t lane = 0; lane < B; ++lane) {
    stepped[(size_t)lane] = mask[lane] && episodes_left[lane] > 0;
    if (!stepped[(size_t)lane]) continue;
    int32_t head = ens.heads[lane];
    if ((uint32_t)head >= (uint32_t)ens.num_heads) {
      if (e->bad_action_host) *e->bad_action_host = 1;
      head = head < 0 ? 0 : ens.num_heads - 1;
    }
    memcpy(rows.data() + lane * A, ens.values + ((int64_t)head * B + lane) * A, (size_t)A * sizeof(float));
  }
  bsb_policy gathered = policy;
  gathered.values = rows.data();
  if (replay) host_record<V>(e, a, mask, episodes_left, previous, &gathered, *replay);
  else host_policy<V>(e, a, mask, episodes_left, previous, gathered);
  for (int64_t lane = 0; lane < B; ++lane) {
    if (!stepped[(size_t)lane] || episodes_left[lane] == before[(size_t)lane]) continue;
    EnvParams lp = p;                     // the lane's setting: its lane_offset keys the stream as the kernel's does
    if constexpr (V::kRagged) {
      ragged_setting_params(lp, ragged_setting(ragged, lane / ragged->pack.lanes_per_setting), ragged->mapping_bits);
    } else if constexpr (V::kPacked) {
      pack_lane_params(lp, lane);
    }
    ens.heads[lane] = ensemble_head(policy.seed, lp.lane_offset + (uint64_t)lane, (uint64_t)a.step0, ens.num_heads);
  }
}

// Kernels and host path of variant V, the runner bsb_create stores in the handle.  The bit sources and kernels are
// those the variant list (BSB_VARIANTS) compiles for V: bsb_create picks no runner for an MT19937 handle whose variant
// lacks MT19937, and only a variant with two_phase_host_kernel is given `two_phase` (a two-phase host step).
template <class V>
int run_variant(bsb_env* e, const LaunchArgs& a, cudaStream_t stream, const TwoPhaseArgs* two_phase) {
  constexpr bool kMt = Compiled<V>::kMt;
  const bool mt = e->p.rng_kind == BSB_RNG_MT19937;
  if (e->device < 0) { run_host<V>(e, a); return BSB_OK; }
  return with_flags(e, a, [&](auto noise, auto track) {
    constexpr bool kNoise = decltype(noise)::value, kTrack = decltype(track)::value;
    if constexpr (Compiled<V>::kTwoPhase) {
      if (two_phase) {
        if constexpr (kMt) { if (mt) return two_phase_launch<V, 1, kNoise, kTrack>(e, a, *two_phase, stream); }
        return two_phase_launch<V, 0, kNoise, kTrack>(e, a, *two_phase, stream);
      }
    }
    if constexpr (V::kRagged && kNoise) {
      // ragged packs take no reward wrapper (bsb_create_ragged): Logging off / on are their only kernels
      return fail(BSB_INTERNAL, "a ragged pack reached the RewardNoise kernel");
    } else {
      LaunchArgs la = a;
      Geometry g;
      const int rc = plan_launch<typename V::Fam, typename V::Obs, V::kRagged>(e, la, g);
      if (rc != BSB_OK) return rc;
      if constexpr (kMt) { if (mt) return launch(e, la, g, stream, transition_kernel<V, 1, kNoise, kTrack>, e->p, la); }
      return launch(e, la, g, stream, transition_kernel<V, 0, kNoise, kTrack>, e->p, la);
    }
  });
}

// Masked calls of variant V (bsb_reset_masked / bsb_step_masked / bsb_rollout_masked / bsb_step_host_masked /
// bsb_advance_masked): the host path, or one launch of masked_kernel with one chunk of 32 lanes per warp.  A masked
// host step (a launch that carries the mailbox, or a `mask_out` to clear spent lanes in) takes the CALL_HOST
// instantiation; a launch with no observation buffer (bsb_advance_masked) takes CALL_ADVANCE; any other call with
// nothing for the T loop, the action stream or the budgets to do (every masked reset and step) takes CALL_ONE.  A
// budgeted step (`previous` given: bsb_step_budgeted, whose `mask_out` is the mask) takes CALL_BUDGETED, and one with a
// `policy` (bsb_step_budgeted_policy: no actions, the picks to a.actions_out) takes CALL_POLICY.  A budgeted step with
// a `replay` (bsb_step_budgeted_record, actions or a policy) takes CALL_RECORD, and one with a `sequence`
// (bsb_step_budgeted_sequence) takes CALL_SEQUENCE.  An `ensemble` step (bsb_step_budgeted_ensemble: its rule in
// `policy`, a replay optional) takes CALL_ENSEMBLE.
template <class V>
int run_masked(bsb_env* e, const LaunchArgs& a, const uint8_t* mask, int64_t* episodes_left, uint8_t* mask_out,
               const bsb_outputs* previous, const bsb_policy* policy, const bsb_replay* replay,
               const bsb_sequence* sequence, const bsb_ensemble_policy* ensemble, cudaStream_t stream) {
  constexpr bool kMt = Compiled<V>::kMt;
  const bool mt = e->p.rng_kind == BSB_RNG_MT19937;
  if (previous && (a.T != 1 || a.mode != MODE_STEP || !a.actions == !policy || (a.actions_out && !policy) ||
                   a.mailbox || !episodes_left || mask_out != mask))
    return fail(BSB_INTERNAL, "a budgeted step must be one step of the caller's actions or policy, with budgets, "
                              "clearing its mask");
  if (policy && !previous) return fail(BSB_INTERNAL, "a policy step must be a budgeted step");
  if (replay && (!previous || !a.step_type)) return fail(BSB_INTERNAL, "a recorded step must be a budgeted step with step types");
  if (sequence && (!previous || !a.step_type || replay))
    return fail(BSB_INTERNAL, "a sequence step must be a budgeted step with step types and no replay");
  if (ensemble && (!policy || sequence))
    return fail(BSB_INTERNAL, "an ensemble step must be a policy step with no sequence");
  if (e->device < 0) {
    if (ensemble) host_ensemble<V>(e, a, mask_out, episodes_left, previous, *policy, *ensemble, replay);
    else if (sequence) host_sequence<V>(e, a, mask_out, episodes_left, previous, policy, *sequence);
    else if (replay) host_record<V>(e, a, mask_out, episodes_left, previous, policy, *replay);
    else if (policy) host_policy<V>(e, a, mask_out, episodes_left, previous, *policy);
    else if (previous) host_budgeted<V>(e, a, mask_out, episodes_left, previous);
    else run_host<V>(e, a, mask, episodes_left);
    return BSB_OK;
  }
  RecordArgs m;                          // a MaskArgs for every kind but CALL_RECORD and CALL_SEQUENCE
  memset(&m, 0, sizeof(m));
  SequenceArgs sq;                       // CALL_SEQUENCE: m's MaskArgs and the sequence buffers
  memset(&sq, 0, sizeof(sq));
  EnsembleArgs en;                       // CALL_ENSEMBLE: m's RecordArgs and the heads
  memset(&en, 0, sizeof(en));
  m.mask = mask;
  m.noise = e->p.wrapper == BSB_WRAP_REWARD_NOISE ? 1 : 0;
  m.track = e->p.ep != nullptr ? 1 : 0;
  m.episodes_left = episodes_left;
  m.mask_out = mask_out;
  LaunchArgs la = a;
  la.bad_action = e->bad_action_dev;
  la.use_pdl = 0;
  la.work_counter = nullptr;
  Geometry g;
  g.threads = 64;
  g.smem = 0;
  g.n_chunks = launch_chunks(e, V::kRagged, 32);
  g.grid = (g.n_chunks + g.threads / 32 - 1) / (g.threads / 32);
  const bool host_call = a.mailbox || mask_out;
  const bool one_call = a.T == 1 && !episodes_left && !a.actions_out && (a.mode != MODE_STEP || a.actions);
  auto go = [&](auto kind) {
    constexpr int kCall = decltype(kind)::value;
    if constexpr (kCall == CALL_RECORD) {
      if constexpr (kMt) { if (mt) return launch(e, la, g, stream, masked_record_kernel<V, 1>, e->p, la, m); }
      return launch(e, la, g, stream, masked_record_kernel<V, 0>, e->p, la, m);
    } else if constexpr (kCall == CALL_SEQUENCE) {
      if constexpr (kMt) { if (mt) return launch(e, la, g, stream, masked_sequence_kernel<V, 1>, e->p, la, sq); }
      return launch(e, la, g, stream, masked_sequence_kernel<V, 0>, e->p, la, sq);
    } else if constexpr (kCall == CALL_ENSEMBLE) {
      if constexpr (kMt) { if (mt) return launch(e, la, g, stream, masked_ensemble_kernel<V, 1>, e->p, la, en); }
      return launch(e, la, g, stream, masked_ensemble_kernel<V, 0>, e->p, la, en);
    } else {
      const MaskArgs& base = m;
      if constexpr (kMt) { if (mt) return launch(e, la, g, stream, masked_kernel<V, 1, kCall>, e->p, la, base); }
      return launch(e, la, g, stream, masked_kernel<V, 0, kCall>, e->p, la, base);
    }
  };
  if (previous) {
    m.prev_obs = previous->observation;
    m.prev_reward = previous->reward;
    m.prev_reward_f64 = previous->reward_f64;
    m.prev_discount = previous->discount;
    m.prev_step_type = previous->step_type;
    m.prev_final_obs = previous->final_observation;
    m.prev_vec_ok = reinterpret_cast<uintptr_t>(previous->observation) % 16 == 0 ? 1 : 0;
    m.prev_final_vec_ok = reinterpret_cast<uintptr_t>(previous->final_observation) % 16 == 0 ? 1 : 0;
    if (policy) {
      m.policy_values = policy->values;
      m.policy_epsilon = policy->epsilon;
      m.policy_seed = policy->seed;
      m.policy_kind = policy->kind;
    }
    if (replay) {
      m.rec_capacity = replay->capacity;
      m.rec_num_added = replay->num_added;
      m.rec_obs_tm1 = replay->obs_tm1;
      m.rec_action = replay->action;
      m.rec_obs = replay->next.observation;
      m.rec_reward = replay->next.reward;
      m.rec_reward_f64 = replay->next.reward_f64;
      m.rec_discount = replay->next.discount;
      m.rec_step_type = replay->next.step_type;
      m.rec_vec_ok = reinterpret_cast<uintptr_t>(replay->obs_tm1) % 16 == 0 &&
                     reinterpret_cast<uintptr_t>(replay->next.observation) % 16 == 0 &&
                     ((size_t)e->step_elems * (size_t)e->obs_elem_bytes) % 16 == 0 ? 1 : 0;
      if (!ensemble) return go(std::integral_constant<int, CALL_RECORD>());
    }
    if (ensemble) {
      static_cast<RecordArgs&>(en) = m;
      en.ens_heads = ensemble->heads;
      en.ens_num_heads = ensemble->num_heads;
      return go(std::integral_constant<int, CALL_ENSEMBLE>());
    }
    if (sequence) {
      static_cast<MaskArgs&>(sq) = m;
      sq.seq_max_length = sequence->max_length;
      sq.seq_length = sequence->length;
      sq.seq_ready = sequence->ready;
      sq.seq_obs = sequence->observations;
      sq.seq_action = sequence->action;
      sq.seq_reward = sequence->next.reward;
      sq.seq_reward_f64 = sequence->next.reward_f64;
      sq.seq_discount = sequence->next.discount;
      sq.seq_step_type = sequence->next.step_type;
      sq.seq_vec_ok = reinterpret_cast<uintptr_t>(sequence->observations) % 16 == 0 &&
                      ((size_t)e->step_elems * (size_t)e->obs_elem_bytes) % 16 == 0 ? 1 : 0;
      return go(std::integral_constant<int, CALL_SEQUENCE>());
    }
    if (policy) return go(std::integral_constant<int, CALL_POLICY>());
    return go(std::integral_constant<int, CALL_BUDGETED>());
  }
  if (host_call) {
    if (a.T != 1 || a.mode != MODE_STEP || !a.actions || a.actions_out)
      return fail(BSB_INTERNAL, "a masked host step must be one step of the caller's actions");
    return go(std::integral_constant<int, CALL_HOST>());
  }
  if (!a.obs) {
    if (a.mode != MODE_STEP || a.actions || a.actions_out || a.final_obs || a.reward || a.reward_f64 || a.discount ||
        a.step_type)
      return fail(BSB_INTERNAL, "a launch without observations must be an advance: sampled actions, no outputs");
    return go(std::integral_constant<int, CALL_ADVANCE>());
  }
  return one_call ? go(std::integral_constant<int, CALL_ONE>()) : go(std::integral_constant<int, CALL_ROLLOUT>());
}

}  // namespace bsb
