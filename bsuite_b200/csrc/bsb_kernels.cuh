// Fused transition kernels: one per kernel variant (template V: family, observation type, auto-reset mode), specialised
// on the bit source (Philox / MT19937), on whether the RewardNoise wrapper stream
// is live, and on whether the Logging accumulators are tracked.
//
// Thread = lane for the scalar transition (state word(s), action, reward,
// discount, step_type are coalesced 4/8-byte accesses).  Observations are dense
// float32 tensors that must be written fresh every step (the reference allocates
// a new array per step: deep_sea.py:104, catch.py:114); they are the HBM traffic
// that bounds the kernel and are emitted WARP-COOPERATIVELY:
//
//   * row families ((1,k) vectors): each thread renders its row into a per-warp
//     shared-memory stage (double buffered); the warp's [32, k] block is
//     contiguous in global memory, so one elected lane sends it with a single TMA
//     bulk store (cp.async.bulk shared::cta -> global).
//   * catch: the same stage holds the warp's 32 boards and stays ZERO between
//     steps; each thread only un-pokes its two old cells and pokes its two new
//     ones before the elected lane issues the bulk store of all 32 boards.
//   * deep_sea (N x N one-hot tile per lane, 4 KB at N = 32): per warp two staging buffers of m zeroed tiles
//     (m = 8 at N = 32); the threads of a group poke their lanes' hot cells (un-poking what they poked into that
//     buffer two stores ago) and the elected lane issues ONE bulk store of the m contiguous tiles (32 KB).
//     Large stores matter: the TMA unit pays a fixed cost per operation, which 4 KB stores cannot amortise
//     and 32 KB stores can.  Unaligned tiles (odd N) use 16-byte streaming
//     stores instead: the warp walks its lanes, every thread writes part of each lane's tile, the hot cell
//     chosen per float4 from a descriptor broadcast by __shfl_sync.  Tiles in compressible memory (bsb_obs_malloc)
//     of a single-step launch that fills the GPU are compared, not written: the warp reads each tile (cp.async into a
//     small ring in shared memory) and stores only the 128-byte lines that differ from the new observation -- two
//     per tile when the destination holds an earlier observation, as a reused output buffer does.  A destination
//     holding anything else falls back to the streaming stores after a 512-byte probe of the chunk's first tile.
//   * mnist: groups of 4 gathered int8 images -> float32 tiles in shared memory -> one bulk store; the all-zero
//     LAST frames of a group leave as one bulk store from zero tiles the CTA's warps share.
//
// A launch of transition_kernel covers T consecutive steps with lane state held in registers (T = 1 for bsb_step);
// actions come from the caller or from the on-device Philox action stream.  Host-driven steps (bsb_step_host) signal
// completion through a pinned mailbox.  For deep_sea and catch with observations of 1 KB or more they run in two
// phases in a kernel of their own, two_phase_host_kernel (all transitions first, the scalars shipped to the host by a
// few copier blocks, then the observations).  Both kernels share the emitters, the lane open / step / close sequence
// (which the host path runs too) and the completion word.  With use_pdl a kernel is launched with programmatic
// stream serialization: everything before griddepcontrol.wait (index math, zeroing the shared-memory stages)
// overlaps the tail of the previous step's kernel.
// Both kernels take a Variant (below) as their first template argument, e.g. transition_kernel<Variant<DeepSea, float,
// NEXT_STEP>, 0, false, true>: the family, the observation element type and the auto-reset mode.  Observations may be
// written as bfloat16 or uint8 instead of float32 (bsb_config.obs_dtype): the emitters stage and store elements of
// that type, each the float32 value converted by obs_cast (bsb_obs_dtype.h).  Same-step handles
// (BSB_FLAG_SAME_STEP_RESET) reset a lane in the call whose step returned LAST (lane_step) and can emit that LAST's
// observation as well (emit_final).
#pragma once
#include "bsb_families.cuh"

namespace bsb {

// Scalar outputs of one step (null members are skipped): the caller's buffers, or the two-phase host step's device
// staging of them.
struct MailFields {
  float* reward; double* reward_f64; float* discount; int32_t* step_type;
};

struct LaunchArgs {
  const int32_t* actions;   // [T,B] or null (sample on device)
  int32_t* actions_out;     // [T,B] or null
  float* obs;               // [T,B,K]
  float* reward;            // [T,B] or null
  double* reward_f64;       // [T,B] or null
  float* discount;          // [T,B] or null
  int32_t* step_type;       // [T,B] or null
  int64_t T;
  int64_t step0;            // global index of the first step of this launch
  uint64_t action_seed;
  int32_t mode;             // 0 = step, 1 = reset every lane, 2 = constructor init
  int32_t obs_vec_ok;       // obs base and per-step stride are 16-byte aligned
  int32_t emit_bulk;        // use TMA bulk stores where the emitter supports them
  int32_t emit_reuse;       // one-hot tiles without bulk stores: store only the words that differ (emit_onehot_reuse)
  int32_t use_pdl;          // launched with programmatic stream serialization
  int32_t group_lanes;      // deep_sea bulk path: lanes per bulk store (power of two, 1..32)
  int32_t final_vec_ok;     // same-step handles: final_obs base and per-step stride are 16-byte aligned
  unsigned long long* work_counter;  // persistent launches: monotonically increasing chunk counter (device)
  unsigned long long work_base;      // value of *work_counter at which this launch's chunk 0 starts
  // Device clock (graph-safe mode, see the kernel): {steps advanced in this mode, chunk counter, finished CTAs}.
  // Null in the default mode, where `step0` / `work_base` arrive as launch arguments from the host's counters.
  unsigned long long* clock;
  int32_t chunk_lanes;      // lanes per chunk (= per warp pass): 32, or 16 / 8 when the batch would under-fill the SMs
  int32_t stage_rows;       // row / board emitters: number of [32, K] shared-memory stages per warp (2: double buffered;
                            // 1: long rows, where a second stage would cost resident warps; 0: straight to global memory)
  int32_t cta_extra_elems;  // observation elements of shared memory after the per-warp stages (mnist bulk path: the
                            // CTA's all-zero tiles)
  // Host-driven steps (bsb_step_host, pinned buffers): completion is signalled through a pinned mailbox.
  struct HostMailbox* mailbox;       // pinned host memory, device alias (null: ordinary launch).  The last CTA to
                                     // finish stores `done = ticket` there: the host spins on it instead of
                                     // paying a stream synchronise.
  struct DeviceMail* mail;           // device memory: finished-CTA counter and two-phase flags
  unsigned long long ticket;
  int32_t timing;                    // BSB_HOST_TIMING: leave %globaltimer stamps in the mailbox
  float* final_obs;         // same-step handles: [T,B,K] observations of the LAST timesteps (bsb_outputs.final_observation),
                            // or null (always null for host steps)
  int32_t* bad_action;      // pinned host flag (device alias): set to 1 when an action is outside [0, num_actions)
};

// The arguments only two_phase_host_kernel takes.
struct TwoPhaseArgs {
  int32_t copiers;          // blocks [0, copiers) own no chunks at first: they ship the scalars to the host (see the kernel)
  MailFields stage;         // device staging of reward / reward_f64 / discount / step_type
};

// Pinned host memory the host-step kernels signal through.  The last block to finish stores `done = ticket` after a
// system-scope fence, so every output written to host memory (reward / discount / step_type, zero-copy) is visible
// when the host sees it.
struct HostMailbox {
  volatile unsigned long long done;     unsigned long long pad[7];      // device -> host, a line of its own
  // BSB_HOST_TIMING=1 (tools/e2e_timeline.py): %globaltimer stamps of the latest two-phase launch, written by its
  // signaller before `done`: [0] block 0 past the dependency wait, [1] phase 1 complete on every block, [2] just
  // before `done`, [3] the latest exit of any block of the PREVIOUS launch
  volatile unsigned long long stamp[8];
};
struct DeviceMail {
  unsigned long long last_exit;           // BSB_HOST_TIMING: max %globaltimer at which a block of the latest launch left
  unsigned long long finished;            // blocks of the current launch that have finished (phase 1, if two-phase)
  volatile unsigned long long phase1;     // ticket of the latest two-phase launch whose phase 1 is complete
  unsigned long long copied;              // copier blocks of the current two-phase launch that have shipped their share
};

enum { MODE_STEP = 0, MODE_RESET = 1, MODE_INIT = 2 };

// ----- kernel variants --------------------------------------------------------------------------------------------
// The first template argument of both kernels and of the host path: the family, the observation element type O
// (bsb_config.obs_dtype: float, Bf16 or uint8_t; the emitters stage and store elements of that type) and the
// auto-reset mode.  NEXT_STEP: bsb_create.  SAME_STEP (BSB_FLAG_SAME_STEP_RESET): a lane whose step returned LAST is
// reset in the same call (lane_step), and that LAST's observation can be emitted as well (emit_final).  PACKED
// (bsb_create_packed): every lane runs with its setting's parameters (pack_lane_params), found once per launch.
// RAGGED (bsb_create_ragged): a pack whose settings differ in observation shape; chunks never straddle settings
// (ragged_chunks).
enum { NEXT_STEP = 0, SAME_STEP = 1, PACKED = 2, RAGGED = 3 };
template <class Family, class O, int kMode> struct Variant {
  typedef Family Fam;
  typedef O Obs;
  static const bool kSameStep = kMode == SAME_STEP;
  static const bool kPacked = kMode == PACKED;
  static const bool kRagged = kMode == RAGGED;
};

// Every compiled variant, X(family, O, mode, mt, two_phase), by the translation unit that holds its kernels and host
// path: build.py compiles bsb_variants.cu once per BSB_UNIT_<unit> below.  `mt`: MT19937 is compiled beside Philox
// (float32 next-step only).  `two_phase`: two_phase_host_kernel is compiled beside transition_kernel (deep_sea and
// catch, whose observations are rendered from the stored lane state, next-step).  Units: fam_ float32 next-step,
// obs_ reduced dtypes (uint8 only for the 0 / 1 observations of deep_sea and catch), ss_ same-step, pk_ packed (all
// but deep_sea, whose settings differ in observation shape), rg_ ragged packs (the three families whose settings
// differ in observation shape); a handle loads only the modules of its own unit.
#define BSB_UNIT_fam_deep_sea(X) X(DeepSea, float, NEXT_STEP, 1, 1)
#define BSB_UNIT_fam_catch(X) X(Catch, float, NEXT_STEP, 1, 1)
#define BSB_UNIT_fam_cartpole(X) X(Cartpole, float, NEXT_STEP, 1, 0)
#define BSB_UNIT_fam_cartpole_swingup(X) X(CartpoleSwingup, float, NEXT_STEP, 1, 0)
#define BSB_UNIT_fam_mountain_car(X) X(MountainCar, float, NEXT_STEP, 1, 0)
#define BSB_UNIT_fam_memory_chain(X) X(MemoryChain, float, NEXT_STEP, 1, 0)
#define BSB_UNIT_fam_bandit(X) X(Bandit, float, NEXT_STEP, 1, 0)
#define BSB_UNIT_fam_umbrella_chain(X) X(UmbrellaChain, float, NEXT_STEP, 1, 0)
#define BSB_UNIT_fam_discounting_chain(X) X(DiscountingChain, float, NEXT_STEP, 1, 0)
#define BSB_UNIT_fam_mnist(X) X(Mnist, float, NEXT_STEP, 1, 0)
#define BSB_UNIT_obs_deep_sea(X) X(DeepSea, Bf16, NEXT_STEP, 0, 1) X(DeepSea, uint8_t, NEXT_STEP, 0, 1)
#define BSB_UNIT_obs_catch(X) X(Catch, Bf16, NEXT_STEP, 0, 1) X(Catch, uint8_t, NEXT_STEP, 0, 1)
#define BSB_UNIT_obs_cartpole(X) X(Cartpole, Bf16, NEXT_STEP, 0, 0)
#define BSB_UNIT_obs_cartpole_swingup(X) X(CartpoleSwingup, Bf16, NEXT_STEP, 0, 0)
#define BSB_UNIT_obs_mountain_car(X) X(MountainCar, Bf16, NEXT_STEP, 0, 0)
#define BSB_UNIT_obs_memory_chain(X) X(MemoryChain, Bf16, NEXT_STEP, 0, 0)
#define BSB_UNIT_obs_bandit(X) X(Bandit, Bf16, NEXT_STEP, 0, 0)
#define BSB_UNIT_obs_umbrella_chain(X) X(UmbrellaChain, Bf16, NEXT_STEP, 0, 0)
#define BSB_UNIT_obs_discounting_chain(X) X(DiscountingChain, Bf16, NEXT_STEP, 0, 0)
#define BSB_UNIT_obs_mnist(X) X(Mnist, Bf16, NEXT_STEP, 0, 0)
#define BSB_UNIT_ss_deep_sea(X) X(DeepSea, float, SAME_STEP, 0, 0) X(DeepSea, Bf16, SAME_STEP, 0, 0) X(DeepSea, uint8_t, SAME_STEP, 0, 0)
#define BSB_UNIT_ss_catch(X) X(Catch, float, SAME_STEP, 0, 0) X(Catch, Bf16, SAME_STEP, 0, 0) X(Catch, uint8_t, SAME_STEP, 0, 0)
#define BSB_UNIT_ss_cartpole(X) X(Cartpole, float, SAME_STEP, 0, 0) X(Cartpole, Bf16, SAME_STEP, 0, 0)
#define BSB_UNIT_ss_cartpole_swingup(X) X(CartpoleSwingup, float, SAME_STEP, 0, 0) X(CartpoleSwingup, Bf16, SAME_STEP, 0, 0)
#define BSB_UNIT_ss_mountain_car(X) X(MountainCar, float, SAME_STEP, 0, 0) X(MountainCar, Bf16, SAME_STEP, 0, 0)
#define BSB_UNIT_ss_memory_chain(X) X(MemoryChain, float, SAME_STEP, 0, 0) X(MemoryChain, Bf16, SAME_STEP, 0, 0)
#define BSB_UNIT_ss_bandit(X) X(Bandit, float, SAME_STEP, 0, 0) X(Bandit, Bf16, SAME_STEP, 0, 0)
#define BSB_UNIT_ss_umbrella_chain(X) X(UmbrellaChain, float, SAME_STEP, 0, 0) X(UmbrellaChain, Bf16, SAME_STEP, 0, 0)
#define BSB_UNIT_ss_discounting_chain(X) X(DiscountingChain, float, SAME_STEP, 0, 0) X(DiscountingChain, Bf16, SAME_STEP, 0, 0)
#define BSB_UNIT_ss_mnist(X) X(Mnist, float, SAME_STEP, 0, 0) X(Mnist, Bf16, SAME_STEP, 0, 0)
#define BSB_UNIT_pk_catch(X) X(Catch, float, PACKED, 0, 0)
#define BSB_UNIT_pk_cartpole(X) X(Cartpole, float, PACKED, 0, 0)
#define BSB_UNIT_pk_cartpole_swingup(X) X(CartpoleSwingup, float, PACKED, 0, 0)
#define BSB_UNIT_pk_mountain_car(X) X(MountainCar, float, PACKED, 0, 0)
#define BSB_UNIT_pk_memory_chain(X) X(MemoryChain, float, PACKED, 0, 0)
#define BSB_UNIT_pk_bandit(X) X(Bandit, float, PACKED, 0, 0)
#define BSB_UNIT_pk_umbrella_chain(X) X(UmbrellaChain, float, PACKED, 0, 0)
#define BSB_UNIT_pk_discounting_chain(X) X(DiscountingChain, float, PACKED, 0, 0)
#define BSB_UNIT_pk_mnist(X) X(Mnist, float, PACKED, 0, 0)
#define BSB_UNIT_rg_deep_sea(X) X(DeepSea, float, RAGGED, 0, 0)
#define BSB_UNIT_rg_memory_chain(X) X(MemoryChain, float, RAGGED, 0, 0)
#define BSB_UNIT_rg_umbrella_chain(X) X(UmbrellaChain, float, RAGGED, 0, 0)
#define BSB_VARIANTS(X)                                                                                                \
  BSB_UNIT_fam_deep_sea(X) BSB_UNIT_fam_catch(X) BSB_UNIT_fam_cartpole(X) BSB_UNIT_fam_cartpole_swingup(X)             \
  BSB_UNIT_fam_mountain_car(X) BSB_UNIT_fam_memory_chain(X) BSB_UNIT_fam_bandit(X) BSB_UNIT_fam_umbrella_chain(X)      \
  BSB_UNIT_fam_discounting_chain(X) BSB_UNIT_fam_mnist(X)                                                              \
  BSB_UNIT_obs_deep_sea(X) BSB_UNIT_obs_catch(X) BSB_UNIT_obs_cartpole(X) BSB_UNIT_obs_cartpole_swingup(X)             \
  BSB_UNIT_obs_mountain_car(X) BSB_UNIT_obs_memory_chain(X) BSB_UNIT_obs_bandit(X) BSB_UNIT_obs_umbrella_chain(X)      \
  BSB_UNIT_obs_discounting_chain(X) BSB_UNIT_obs_mnist(X)                                                              \
  BSB_UNIT_ss_deep_sea(X) BSB_UNIT_ss_catch(X) BSB_UNIT_ss_cartpole(X) BSB_UNIT_ss_cartpole_swingup(X)                 \
  BSB_UNIT_ss_mountain_car(X) BSB_UNIT_ss_memory_chain(X) BSB_UNIT_ss_bandit(X) BSB_UNIT_ss_umbrella_chain(X)          \
  BSB_UNIT_ss_discounting_chain(X) BSB_UNIT_ss_mnist(X)                                                                \
  BSB_UNIT_pk_catch(X) BSB_UNIT_pk_cartpole(X) BSB_UNIT_pk_cartpole_swingup(X) BSB_UNIT_pk_mountain_car(X)             \
  BSB_UNIT_pk_memory_chain(X) BSB_UNIT_pk_bandit(X) BSB_UNIT_pk_umbrella_chain(X) BSB_UNIT_pk_discounting_chain(X)     \
  BSB_UNIT_pk_mnist(X) BSB_UNIT_rg_deep_sea(X) BSB_UNIT_rg_memory_chain(X) BSB_UNIT_rg_umbrella_chain(X)

// The list's flags of variant V (undefined for a variant the list does not compile).
template <class V> struct Compiled;
#define BSB_COMPILED(F, O, mode, mt, two_phase) \
  template <> struct Compiled<Variant<F, O, mode> > { static const bool kMt = mt, kTwoPhase = two_phase; };
BSB_VARIANTS(BSB_COMPILED)
#undef BSB_COMPILED

// log2 of the observation elements per 16-byte vector store.
template <class O> struct Vec16 { static const int shift = sizeof(O) == 4 ? 2 : sizeof(O) == 2 ? 3 : 4; };

// ----- RNG plumbing ---------------------------------------------------------
template <int RK> struct RngOf;
template <> struct RngOf<0> { typedef LegacyRng<PhiloxSrc> type; };
template <> struct RngOf<1> { typedef LegacyRng<MtSrc> type; };

BSB_HD void rng_open(LegacyRng<PhiloxSrc>& r, const EnvParams& p, int64_t i, bool wrapper) {
  const uint64_t packed = wrapper ? p.wrng_pos[i] : p.rng_pos[i];
  r.src.open(p.seed, p.lane_offset + (uint64_t)i, wrapper ? STREAM_WRAPPER : STREAM_ENV, packed);
  r.g.has = (packed & RNG_HASGAUSS) ? 1 : 0;
  const double* gz = wrapper ? p.wrng_gauss : p.rng_gauss;
  r.g.value = (r.g.has && gz) ? gz[i] : 0.0;
}
BSB_HD void rng_close(const LegacyRng<PhiloxSrc>& r, const EnvParams& p, int64_t i, bool wrapper) {
  const uint64_t packed = r.src.packed() | (r.g.has ? RNG_HASGAUSS : 0ull);
  if (wrapper) p.wrng_pos[i] = packed; else p.rng_pos[i] = packed;
  double* gz = wrapper ? p.wrng_gauss : p.rng_gauss;
  if (gz && r.g.has) gz[i] = r.g.value;
}
BSB_HD void rng_open(LegacyRng<MtSrc>& r, const EnvParams& p, int64_t i, bool wrapper) {
  const int64_t stride = (p.batch > 0) ? p.batch : 1;
  r.src.open((wrapper ? p.wmt_key : p.mt_key) + i, stride, (wrapper ? p.wmt_idx : p.mt_idx)[i]);
  const uint64_t packed = wrapper ? p.wrng_pos[i] : p.rng_pos[i];
  r.g.has = (packed & RNG_HASGAUSS) ? 1 : 0;
  const double* gz = wrapper ? p.wrng_gauss : p.rng_gauss;
  r.g.value = (r.g.has && gz) ? gz[i] : 0.0;
}
BSB_HD void rng_close(const LegacyRng<MtSrc>& r, const EnvParams& p, int64_t i, bool wrapper) {
  (wrapper ? p.wmt_idx : p.mt_idx)[i] = r.src.idx;
  const uint64_t packed = r.g.has ? RNG_HASGAUSS : 0ull;
  if (wrapper) p.wrng_pos[i] = packed; else p.rng_pos[i] = packed;
  double* gz = wrapper ? p.wrng_gauss : p.rng_gauss;
  if (gz && r.g.has) gz[i] = r.g.value;
}

// ----- the per-lane call sequence of base.Environment.step (base.py:59-65) --
// followed by the reward wrappers (utils/wrappers.py:275-283, 338-346), which
// act on every non-FIRST timestep; bsuite_info() stays un-noised / un-scaled.
template <class F, class R, class WR>
BSB_HD StepOut lane_transition(const EnvParams& p, int64_t i, typename F::Lane& L, R& rng, WR& wrng,
                               int32_t action, int32_t mode, bool noise) {
  StepOut o;
  if (mode == MODE_RESET || L.nr) {        // `if self._reset_next_step: return self.reset()`
    o = F::reset(p, i, L, rng);
    L.nr = 0;
  } else {
    o = F::step(p, i, L, action, rng);
    L.nr = (o.step_type == LAST) ? 1u : 0u;
    if (noise) { o.reward = o.reward + p.noise_scale * wrng.randn(); }
    else if (p.wrapper == 2) { o.reward = o.reward * p.reward_scale; }
  }
  return o;
}

// ----- one lane over a run of steps: open, one lane_step per step, close ------------------------------------------
// The kernels and the host path (host_run) all go through these three.  Reading and checking the action stays with
// each caller: the host path rejects bad actions up front, the kernels clamp them and raise `bad_action`.
// Opens the lane's state (F::init for the constructor), both RNG streams and the Logging accumulators.
// `state_loaded`: the caller has read L and ep already (phase 1 of the two-phase host step batches those loads).
template <class F, class R>
BSB_HD void lane_open(const EnvParams& p, int64_t lane, typename F::Lane& L, R& rng, R& wrng, EpisodeStats& ep,
                      int32_t mode, bool noise, bool track, bool state_loaded = false) {
  if (!state_loaded) { if (mode == MODE_INIT) F::init(p, L); else F::load(p, lane, L); }
  if (p.rng_pos) rng_open(rng, p, lane, false);
  if (noise) rng_open(wrng, p, lane, true);
  if (track && !state_loaded) ep.load(p, lane);
}
template <class F, class R>
BSB_HD void lane_close(const EnvParams& p, int64_t lane, const typename F::Lane& L, const R& rng, const R& wrng,
                       const EpisodeStats& ep, bool noise, bool track) {
  F::store(p, lane, L);
  if (p.rng_pos) rng_close(rng, p, lane, false);
  if (noise) rng_close(wrng, p, lane, true);
  if (track) ep.store(p, lane);
}
// Random draws an observation makes while it is rendered: umbrella_chain's distractors (umbrella_chain.py:60-66),
// drawn exactly as UmbrellaChain::row draws them.  Every other observation is a function of the lane state.
template <class F> struct ObsDraws { template <class R> static BSB_HD void skip(const EnvParams&, R&) {} };
template <> struct ObsDraws<UmbrellaChain> {
  template <class R> static BSB_HD void skip(const EnvParams& p, R& rng) {
    for (int k0 = 0; k0 < p.n_distractor; k0 += 64) rng.binomial_half_bits((p.n_distractor - k0) < 64 ? (p.n_distractor - k0) : 64);
  }
};
// Same-step auto-reset: a step that returns LAST runs the family's reset in the same call.  The reference's order of
// draws for the two calls folded together is kept: the step's, the LAST observation's (skipped here, replayed from
// `rng` when the final observation is rendered), the reset's, the FIRST observation's.
template <class F, class R> struct MergedReset {
  typename F::Lane last;   // the lane at the LAST, before the reset: the final observation is rendered from it
  R rng;                   // the env stream before the LAST observation's draws
  bool done;               // this call returned LAST and reset the lane
};

// One step of an open lane: the transition, the Logging accumulators with their log row, and the four scalar outputs
// at index `off` of `out` (null outputs are skipped).  `step`: global index of this step.
// kSameStep: `merged` receives the lane as it was at a LAST, and the lane is reset in the same call.  The Logging
// columns episode_len / episode_return restart at the NEXT call, which the marker ep[5] (same-step handles only)
// announces: the lane's _reset_next_step bit, which next-step handles use, is clear again after a merged reset.
template <class F, class R, bool kSameStep = false>
BSB_HD void lane_step(const EnvParams& p, int64_t lane, typename F::Lane& L, R& rng, R& wrng, EpisodeStats& ep,
                      int32_t action, int32_t mode, bool noise, bool track, int64_t step, const MailFields& out,
                      int64_t off, MergedReset<F, R>* merged = nullptr) {
  bool after_last = L.nr != 0;
  const StepOut o = lane_transition<F, R, R>(p, lane, L, rng, wrng, action, mode, noise);
  if (track) {
    if constexpr (kSameStep) {
      double* restart = p.ep + 5 * p.batch + lane;
      if (*restart != 0.0) {                 // the first call since a merged reset
        *restart = 0.0;
        if (o.step_type == FIRST) after_last = true;          // an explicit reset: as after a LAST
        else { ep.episode_return = 0.0; p.ep[4 * p.batch + lane] = (double)(step - 1); }   // the episode began at the merged call
      }
    }
    ep.track(p, lane, o, step, after_last);
    if (p.log_rows && o.step_type == LAST && log_row_due(p, lane)) {      // <= 49 times per 10 000 episodes
      F::store(p, lane, L); ep.store(p, lane);                          // the row reads them from memory
      log_row_write(p, lane, step + 1);
    }
  }
  if (out.reward) out.reward[off] = (float)o.reward;
  if (out.reward_f64) out.reward_f64[off] = o.reward;
  if (out.discount) out.discount[off] = o.discount;
  if (out.step_type) out.step_type[off] = o.step_type;
  if constexpr (kSameStep) {
    merged->done = o.step_type == LAST;
    if (merged->done) {
      merged->last = L;
      merged->rng = rng;
      ObsDraws<F>::skip(p, rng);
      F::reset(p, lane, L, rng);
      L.nr = 0;
      if (track) p.ep[5 * p.batch + lane] = 1.0;
    }
  }
}

// A lane that sits out a masked call (bsb_step_masked / bsb_reset_masked, or a step of bsb_rollout_masked) makes no
// call, but the handle's call count still advances, and episode_stat / log_row_write read the lane's Logging columns
// from that global count.  So the lane's own counters move instead: first_count and start_call each gain the skipped
// call, and steps = calls - first_count and episode_len = calls - 1 - start_call keep the values of the lane's own call
// sequence.  Before the lane's first call (first_count == 0 means "no episode yet" to episode_len) the first skip sets
// first_count to 1 and leaves start_call at 0: after d skips first_count = d and start_call = d - 1, which read steps =
// episode_len = 0, and the lane's first call overwrites start_call (it follows the constructor's _reset_next_step, as
// after a LAST).  The same-step marker ep[5] waits for the lane's next call and is left alone.
// d >= 1 consecutive sit-outs at once (a masked rollout's sit-outs all follow the lane's last active call):
// first_count gains d, start_call d, or d - 1 when the first of them met first_count == 0.
BSB_HD void lane_sit_out_calls(const EnvParams& p, int64_t lane, int64_t d) {
  double* first_count = p.ep + 3 * p.batch + lane;
  double* start_call = p.ep + 4 * p.batch + lane;
  *start_call += (double)(*first_count != 0.0 ? d : d - 1);
  *first_count += (double)d;
}

// Observation emitter of each family.
static const int EMIT_ROWS = 0, EMIT_ONEHOT = 1, EMIT_TWOHOT = 2, EMIT_IMAGE = 3;
// Families whose observation is a pure function of the STORED lane state (F::describe after F::load): their
// host-driven steps can deliver the scalars before the observation is streamed (two-phase host step).
template <class F> struct ObsFromState { static const bool value = false; };
template <> struct ObsFromState<DeepSea> { static const bool value = true; };
template <> struct ObsFromState<Catch> { static const bool value = true; };
template <class F> struct EmitKind { static const int value = EMIT_ROWS; };
template <> struct EmitKind<DeepSea> { static const int value = EMIT_ONEHOT; };
template <> struct EmitKind<Catch> { static const int value = EMIT_TWOHOT; };
template <> struct EmitKind<Mnist> { static const int value = EMIT_IMAGE; };
static const int ROW_STAGES = 2;      // at most: double-buffered [32, K] stage per warp (LaunchArgs::stage_rows)
static const int TILE_STAGES = 2;     // deep_sea bulk path: double-buffered groups of `group_lanes` tiles per warp
static const int REUSE_WORDS = 256;   // compare-then-store tiles: 16-byte words per pass (8 per thread) ...
static const int REUSE_STAGES = 2;    // ... and passes in flight per warp (emit_onehot_reuse)
static const int REUSE_STORE_WORDS = 8;   // ... and a differing word is stored with its whole 128-byte line

// Dynamic shared memory per warp, in observation elements of type O (times sizeof(O): bytes).
template <class F, class O> inline
#if defined(__CUDACC__)
__host__ __device__
#endif
size_t smem_elems_per_warp(int K, bool emit_bulk, bool emit_reuse, int group_lanes, int row_stages) {
  if (EmitKind<F>::value == EMIT_ROWS || EmitKind<F>::value == EMIT_TWOHOT) return (size_t)row_stages * 32 * (size_t)K;
  if (EmitKind<F>::value == EMIT_ONEHOT && emit_bulk) return (size_t)TILE_STAGES * (size_t)group_lanes * (size_t)K;
  if (EmitKind<F>::value == EMIT_ONEHOT && emit_reuse) return (size_t)REUSE_STAGES * REUSE_WORDS * 16 / sizeof(O);
  if (EmitKind<F>::value == EMIT_IMAGE)                    // int8 pixel -> float32 table (+ one staging buffer of m tiles)
    return 256 * sizeof(float) / sizeof(O) + (emit_bulk ? (size_t)group_lanes * (size_t)K : 0);
  return 0;
}

// deep_sea bulk path: lanes per bulk store of tiles of `tile` bytes, the largest power of two <= 16 with one store
// <= 40 KB, so a group never spans a 32-lane chunk.  N = 32 -> 8 lanes (32 KB stores; 88.8 us per headline step
// against 91.9 with 4 lanes, DESIGN.md §3), N = 50 -> 4 lanes (40 KB).  Narrow tiles reach the 16-lane cap first:
// N = 32 in bfloat16 -> 16 lanes (32 KB), in uint8 -> 16 lanes (16 KB).  0: no bulk path, the store is not a whole
// number of 16-byte words or the two staged groups exceed 100 KB.
inline int tile_group_lanes(size_t tile) {
  int m = 1;
  while (m < 16 && (size_t)(2 * m) * tile <= 40 * 1024) m <<= 1;
  return (((size_t)m * tile) % 16 != 0 || (size_t)TILE_STAGES * m * tile > 100 * 1024) ? 0 : m;
}

#if defined(__CUDACC__)

__device__ __forceinline__ void st_stream(float4* dst, float4 v) { __stcs(dst, v); }
__device__ __forceinline__ void st_stream(float* dst, float v) { __stcs(dst, v); }
__device__ __forceinline__ void st_stream(Bf16* dst, Bf16 v) { __stcs(reinterpret_cast<unsigned short*>(dst), v.bits); }
__device__ __forceinline__ void st_stream(uint8_t* dst, uint8_t v) { __stcs(dst, v); }
// Bits of the observation element O for 1.0 (the hot cells of deep_sea and catch).
template <class O> __device__ __forceinline__ uint32_t one_bits() {
  return sizeof(O) == 2 ? 0x3f80u : 1u;       // bfloat16 1.0, uint8 1
}
// Four consecutive observation elements (one 16-, 8- or 4-byte word) from four float32 values.
template <class O> struct Quad;
template <> struct Quad<float> { typedef float4 type; static __device__ __forceinline__ float4 of(float4 v) { return v; } };
template <> struct Quad<Bf16> {
  typedef uint2 type;
  static __device__ __forceinline__ uint2 of(float4 v) {
    return make_uint2((uint32_t)f32_to_bf16_bits(v.x) | ((uint32_t)f32_to_bf16_bits(v.y) << 16),
                      (uint32_t)f32_to_bf16_bits(v.z) | ((uint32_t)f32_to_bf16_bits(v.w) << 16));
  }
};
template <> struct Quad<uint8_t> {
  typedef unsigned int type;
  static __device__ __forceinline__ unsigned int of(float4 v) {
    return (uint32_t)f32_to_u8(v.x) | ((uint32_t)f32_to_u8(v.y) << 8) | ((uint32_t)f32_to_u8(v.z) << 16) |
           ((uint32_t)f32_to_u8(v.w) << 24);
  }
};
__device__ __forceinline__ void st_stream(uint2* dst, uint2 v) { __stcs(dst, v); }
__device__ __forceinline__ void st_stream(unsigned int* dst, unsigned int v) { __stcs(dst, v); }

// ----- TMA bulk store (shared::cta -> global) and PDL primitives --------------
// Bulk store with an L2 eviction-priority hint (policy from createpolicy.fractional.L2::evict_first).
__device__ __forceinline__ void bulk_store_s2g_hint(void* gdst, const void* ssrc, uint32_t bytes, uint64_t policy) {
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(ssrc);
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(gdst), "r"(s), "r"(bytes), "l"(policy) : "memory");
}
// Not volatile: the policy is a pure value, so the compiler may create it once and reuse it across stores.
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
  uint64_t p; asm("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p;
}
// Observation bulk store: observations are written once and never re-read by this kernel, so they are marked
// evict_first (DESIGN.md §3 records the H100 A/B against the other policies).
__device__ __forceinline__ void bulk_store_obs(void* gdst, const void* ssrc, uint32_t bytes) {
  bulk_store_s2g_hint(gdst, ssrc, bytes, l2_policy_evict_first());
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ----- vector-store emitters ---------------------------------------------------
// One-hot tiles: `hot` is the flat index of the single 1.0 (or -1: all zeros).  `vec`: 16-byte stores (every tile
// is a whole number of them).
template <class O>
__device__ __forceinline__ void emit_onehot_vec(O* obs_t, int64_t warp_base, int n_lanes, int K, int hot, bool vec) {
  const int tid = threadIdx.x & 31;
  if (vec && sizeof(O) != 4) {
    // 8 bfloat16 or 16 uint8 per store: the hot element is one word of the store's four, shifted into place
    constexpr int S = Vec16<O>::shift;
    const int KV = K >> S;
    for (int j = 0; j < n_lanes; ++j) {
      const int h = __shfl_sync(0xffffffffu, hot, j);
      const int hq = h < 0 ? -1 : (h >> S), hb = (h & ((1 << S) - 1)) * (int)sizeof(O);
      const int word = hb >> 2;
      const uint32_t bits = one_bits<O>() << ((hb & 3) * 8);
      uint4* dst = reinterpret_cast<uint4*>(obs_t + (warp_base + j) * (int64_t)K);
#pragma unroll 8
      for (int q = tid; q < KV; q += 32) {
        uint4 v = make_uint4(0u, 0u, 0u, 0u);
        if (q == hq) { if (word == 0) v.x = bits; else if (word == 1) v.y = bits; else if (word == 2) v.z = bits; else v.w = bits; }
        __stcs(dst + q, v);
      }
    }
  } else if (vec) {
    const int K4 = K >> 2;
    for (int j = 0; j < n_lanes; ++j) {
      const int h = __shfl_sync(0xffffffffu, hot, j);
      const int hq = h >> 2, hc = h & 3;
      float4* dst = reinterpret_cast<float4*>(obs_t + (warp_base + j) * (int64_t)K);
#pragma unroll 8
      for (int q = tid; q < K4; q += 32) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (q == hq) { if (hc == 0) v.x = 1.f; else if (hc == 1) v.y = 1.f; else if (hc == 2) v.z = 1.f; else v.w = 1.f; }
        st_stream(dst + q, v);
      }
    }
  } else {
    for (int j = 0; j < n_lanes; ++j) {
      const int h = __shfl_sync(0xffffffffu, hot, j);
      O* dst = obs_t + (warp_base + j) * (int64_t)K;
      for (int e = tid; e < K; e += 32) st_stream(dst + e, obs_cast<O>(e == h ? 1.f : 0.f));
    }
  }
}

// Compare-then-store one-hot tiles (LaunchArgs::emit_reuse; every tile a whole number of 16-byte words): the warp
// reads each tile and stores only the 128-byte lines that hold a word whose bits differ from the word this step
// produces, so a destination that already holds an earlier one-hot observation costs a read of the tile and at most
// two line stores (the old hot cell's and the new one's).  Bits are compared, not values, so -0.0 and NaN payloads
// are rewritten: the result is bit-identical to a full write whatever the destination held.  Whole lines, not single
// 16-byte words: a partial store into a line of compressible memory made single steps 1.5x slower than full writes
// (DESIGN.md §7, "Compressible observation memory").
// The tiles are read in PASSES of REUSE_WORDS words (8 per thread; one pass per 4 KB tile) through a ring of
// REUSE_STAGES passes in the warp's shared memory, with cp.async (the loads in flight hold no registers): the next
// pass is always in flight while the current one is compared.  Every thread compares exactly the words it loaded, so
// no warp barrier is needed between the two.
// A destination that does not hold an observation must not pay a read on top of every write.  A PROBE of the first
// 512 bytes of the chunk's first tile decides whether the chunk is read at all; after it, any pass that holds more
// than two differing words turns the rest of the chunk blind: streaming stores of every word, as emit_onehot_vec.
__device__ __forceinline__ void cp_async16(void* sdst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(sdst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// Issues pass s of the chunk's tiles into ring slot s % REUSE_STAGES as one commit group (empty past the last pass).
template <class O>
__device__ __forceinline__ void reuse_load(uint4* ring, const O* obs_t, int64_t warp_base, int n_lanes, int K, int s) {
  const int KV = K >> Vec16<O>::shift;                      // 16-byte words per tile
  const int passes = (KV + REUSE_WORDS - 1) / REUSE_WORDS;
  if (s < n_lanes * passes) {
    const int j = s / passes, q0 = (s - j * passes) * REUSE_WORDS;
    const uint4* src = reinterpret_cast<const uint4*>(obs_t + (warp_base + j) * (int64_t)K) + q0;
    uint4* slot = ring + (s % REUSE_STAGES) * REUSE_WORDS;
    for (int q = threadIdx.x & 31; q < REUSE_WORDS && q0 + q < KV; q += 32) cp_async16(slot + q, src + q);
  }
  cp_async_commit();
}
// What word `q` of a one-hot tile whose hot element is `h` (-1: none) holds: zero, or the hot word.
template <class O>
__device__ __forceinline__ uint4 onehot_word(int h, int q) {
  constexpr int S = Vec16<O>::shift;
  uint4 v = make_uint4(0u, 0u, 0u, 0u);
  if (h >= 0 && q == (h >> S)) {
    const int hb = (h & ((1 << S) - 1)) * (int)sizeof(O), part = hb >> 2;
    const uint32_t bits = (sizeof(O) == 4 ? 0x3f800000u : one_bits<O>()) << ((hb & 3) * 8);
    if (part == 0) v.x = bits; else if (part == 1) v.y = bits; else if (part == 2) v.z = bits; else v.w = bits;
  }
  return v;
}
__device__ __forceinline__ bool bits_differ(uint4 a, uint4 b) { return ((a.x ^ b.x) | (a.y ^ b.y) | (a.z ^ b.z) | (a.w ^ b.w)) != 0u; }
template <class O>
__device__ __forceinline__ void emit_onehot_reuse(uint4* ring, O* obs_t, int64_t warp_base, int n_lanes, int K, int hot) {
  constexpr int S = Vec16<O>::shift;
  const int tid = threadIdx.x & 31;
  const int KV = K >> S;
  const int passes = (KV + REUSE_WORDS - 1) / REUSE_WORDS;
  const int n = n_lanes * passes;
  // The probe: the first 32 words (512 bytes) of the chunk's first tile decide whether the chunk is read at all.
  const int h0 = __shfl_sync(0xffffffffu, hot, 0);
  const uint4* tile0 = reinterpret_cast<const uint4*>(obs_t + warp_base * (int64_t)K);
  if (tid < KV) cp_async16(ring + tid, tile0 + tid);
  cp_async_commit();
  cp_async_wait<0>();
  bool blind = __popc(__ballot_sync(0xffffffffu, tid < KV && bits_differ(ring[tid], onehot_word<O>(h0, tid)))) > 2;
  if (!blind) for (int k = 0; k < REUSE_STAGES; ++k) reuse_load(ring, obs_t, warp_base, n_lanes, K, k);
  for (int s = 0; s < n; ++s) {
    const int j = s / passes, q0 = (s - j * passes) * REUSE_WORDS;
    const int h = __shfl_sync(0xffffffffu, hot, j);
    uint4* dst = reinterpret_cast<uint4*>(obs_t + (warp_base + j) * (int64_t)K) + q0;
    const uint4* slot = ring + (s % REUSE_STAGES) * REUSE_WORDS;
    if (!blind) cp_async_wait<REUSE_STAGES - 1>();           // this thread's words of pass s have landed
    unsigned differing = 0;
#pragma unroll 2
    for (int u = 0; u < REUSE_WORDS / 32 && u * 32 < KV - q0; ++u) {
      const int q = u * 32 + tid;
      const bool in = q0 + q < KV;
      const uint4 v = onehot_word<O>(h, q0 + q);
      const bool differs = in && (blind || bits_differ(slot[q], v));
      const unsigned mask = __ballot_sync(0xffffffffu, differs);
      differing += __popc(mask);
      // a differing word is stored with the rest of its REUSE_STORE_WORDS-word block
      const unsigned block = (unsigned)((1ull << REUSE_STORE_WORDS) - 1ull) << (tid & ~(REUSE_STORE_WORDS - 1));
      if (in && (mask & block) != 0u) __stcs(dst + q, v);
    }
    if (!blind) {
      blind = differing > 2u;
      if (!blind) reuse_load(ring, obs_t, warp_base, n_lanes, K, s + REUSE_STAGES);     // into the slot just compared
    }
  }
  cp_async_wait<0>();                                       // nothing lands in the ring after the emitter returns
}

// Boards with up to two hot cells; the warp's boards form one contiguous span.  Its start is 16-byte aligned
// whenever its length is a whole number of 16-byte stores: a full chunk of 8, 16 or 32 boards of K elements of s
// bytes starts at a multiple of 8 * K * s bytes, which is a multiple of 16 unless s = 1 and K is odd -- and then no
// span of fewer than 16 boards is a multiple of 16 bytes long.
template <class O>
__device__ __forceinline__ void emit_twohot_vec(O* obs_t, int64_t warp_base, int n_lanes, int K, int hot_a, int hot_b, bool vec) {
  const int tid = threadIdx.x & 31;
  const int total = n_lanes * K;
  O* dst = obs_t + warp_base * (int64_t)K;
  constexpr int S = Vec16<O>::shift;
  if (vec && sizeof(O) != 4 && (total & ((1 << S) - 1)) == 0) {
    const int totalV = total >> S;
    for (int q0 = 0; q0 < totalV; q0 += 32) {
      const int q = q0 + tid;
      const int e0 = (q < totalV ? q : 0) << S;
      int j = e0 / K, c = e0 - j * K;
      uint32_t w[4] = {0u, 0u, 0u, 0u};
#pragma unroll
      for (int k = 0; k < (1 << S); ++k) {
        const int jj = j < 32 ? j : 31;
        const int a = __shfl_sync(0xffffffffu, hot_a, jj);
        const int b = __shfl_sync(0xffffffffu, hot_b, jj);
        if (c == a || c == b) w[(k * (int)sizeof(O)) >> 2] |= one_bits<O>() << (((k * (int)sizeof(O)) & 3) * 8);
        if (++c >= K) { c = 0; ++j; }
      }
      if (q < totalV) __stcs(reinterpret_cast<uint4*>(dst) + q, make_uint4(w[0], w[1], w[2], w[3]));
    }
  } else if (vec && (total & ((1 << S) - 1)) == 0) {
    const int total4 = total >> 2;
    for (int q0 = 0; q0 < total4; q0 += 32) {
      const int q = q0 + tid;
      const int e0 = (q < total4 ? q : 0) << 2;
      int j = e0 / K, c = e0 - j * K;
      float v[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int jj = j < 32 ? j : 31;
        const int a = __shfl_sync(0xffffffffu, hot_a, jj);
        const int b = __shfl_sync(0xffffffffu, hot_b, jj);
        v[k] = (c == a || c == b) ? 1.f : 0.f;
        if (++c >= K) { c = 0; ++j; }
      }
      if (q < total4) st_stream(reinterpret_cast<float4*>(dst) + q, make_float4(v[0], v[1], v[2], v[3]));
    }
  } else {
    for (int e0 = 0; e0 < total; e0 += 32) {
      const int e = e0 + tid;
      const int ee = e < total ? e : 0;
      const int j = ee / K, c = ee - j * K;
      const int a = __shfl_sync(0xffffffffu, hot_a, j);
      const int b = __shfl_sync(0xffffffffu, hot_b, j);
      if (e < total) st_stream(dst + e, obs_cast<O>((c == a || c == b) ? 1.f : 0.f));
    }
  }
}

// Image tiles gathered from the int8 dataset (`image` < 0: zeros).  `lut` is the warp's 256-entry table of
// (float)(int8)i / 255 in shared memory: IEEE float division costs ~10 instructions and takes a slow path for zero
// numerators (most MNIST pixels), a table lookup costs one LDS.  The gather is latency-bound if each load ->
// convert -> store chain runs serially, so all loads of a pass (8 x 32 char4 = 1 024 pixels) are issued first.
// Observations of type O other than float32 convert each looked-up float32 (4 pixels: one 8-byte bfloat16 store).
template <class O>
__device__ __forceinline__ void emit_image(const EnvParams& p, const float* lut, O* obs_t, int64_t warp_base, int n_lanes, int K, int image, bool vec) {
  const int tid = threadIdx.x & 31;
  constexpr int U = 8;
  for (int j = 0; j < n_lanes; ++j) {
    const int img = __shfl_sync(0xffffffffu, image, j);
    O* dst = obs_t + (warp_base + j) * (int64_t)K;
    const int8_t* src = p.images + (int64_t)(img < 0 ? 0 : img) * K;
    if (vec) {
      const int K4 = K >> 2;
      const uchar4* src4 = reinterpret_cast<const uchar4*>(src);
      typename Quad<O>::type* dst4 = reinterpret_cast<typename Quad<O>::type*>(dst);
      if (img < 0) {
        for (int q = tid; q < K4; q += 32) st_stream(dst4 + q, Quad<O>::of(make_float4(0.f, 0.f, 0.f, 0.f)));
        continue;
      }
      for (int q0 = 0; q0 < K4; q0 += 32 * U) {
        uchar4 c[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int q = q0 + u * 32 + tid;
          c[u] = make_uchar4(0, 0, 0, 0);
          if (q < K4) c[u] = __ldg(src4 + q);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int q = q0 + u * 32 + tid;
          if (q < K4) st_stream(dst4 + q, Quad<O>::of(make_float4(lut[c[u].x], lut[c[u].y], lut[c[u].z], lut[c[u].w])));
        }
      }
    } else {
      for (int e = tid; e < K; e += 32) st_stream(dst + e, obs_cast<O>(img >= 0 ? lut[(uint8_t)src[e]] : 0.f));
    }
  }
}

// image.astype(float32) / 255 (mnist.py:64) without a table, an IEEE division or an int->float conversion (I2F runs
// on the quarter-rate XU pipe): per pixel one PRMT (sign-extended byte: the reference parses images as INT8,
// utils/datasets.py:55-56), one IADD + one FADD (v as float through the 1.5 * 2^23 magic number, exact for
// |v| <= 128), then the quotient as fma(v, hi, v * lo) with hi + lo = 1/255 split into two floats.  That is the
// correctly rounded v / 255 for every int8 v: checked exhaustively against numpy on the device
// (tests/test_round2_features.py) -- 256 inputs, no reasoning about rounding needed.
__device__ __forceinline__ float pixel_div255(uint32_t word, int byte) {
  // prmt.b32: bit 3 of a selector nibble replicates the sign of the selected byte (the __byte_perm intrinsic masks
  // that bit off): byte `byte` in the low byte, its sign in the three bytes above = the sign-extended int8
  const uint32_t sel = (uint32_t)byte | ((8u | (uint32_t)byte) << 4) | ((8u | (uint32_t)byte) << 8) | ((8u | (uint32_t)byte) << 12);
  int v;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(v) : "r"(word), "r"(0u), "r"(sel));
  const float x = __fadd_rn(__int_as_float(0x4B400000 + v), -12582912.0f);
  const float hi = 0.003921568859368563f, lo = -2.319175823606301e-10f;      // float(1/255), float(1/255 - hi)
  return __fmaf_rn(x, hi, __fmul_rn(x, lo));
}
__device__ __forceinline__ float4 pixels4(uint32_t w) {
  return make_float4(pixel_div255(w, 0), pixel_div255(w, 1), pixel_div255(w, 2), pixel_div255(w, 3));
}

// Image tiles through shared memory and the TMA unit (K % 16 == 0, e.g. 28 x 28).  The chunk's lanes are walked in
// blocks of `mz` consecutive lanes (= mz contiguous tiles in global memory):
//   * a block whose lanes all show the all-zero LAST frame (mnist.py:74; every other step of every lane) is ONE
//     bulk store of mz tiles (25 KB at mz = 8) from the CTA's zero tiles -- nothing is staged, nothing waited for;
//   * otherwise the block goes in groups of `m` (<= 4) lanes: all 16-byte loads of the group's int8 images (49 per
//     28 x 28 tile) are issued before the first conversion, the float32 tiles land in a staging buffer and leave
//     as one bulk store of m * 4K bytes.
// stage = [256 floats: table of the vector path][m x K elements of O; a bfloat16 tile is converted after
// pixel_div255].  One staging buffer per warp (13.25 KB at m = 4 in float32) keeps more warps resident than two --
// the conversion is issue-bound, so resident warps matter -- while the zero frames, which are pure bandwidth, still
// leave in 24.5 KB stores.
template <class O>
__device__ __forceinline__ void emit_image_bulk(const EnvParams& p, O* stage, const O* cta_zero, O* obs_t,
                                                int64_t warp_base, int n_lanes, int K, int image, int m, int mz) {
  constexpr int MAXM = 4;
  const int tid = threadIdx.x & 31;
  O* const buf = reinterpret_cast<O*>(reinterpret_cast<float*>(stage) + 256);
  const int K16 = K >> 4;
  const unsigned showing = __ballot_sync(0xffffffffu, image >= 0);
  for (int z0 = 0; z0 < n_lanes; z0 += mz) {
    const int in_block = (n_lanes - z0) < mz ? (n_lanes - z0) : mz;
    const unsigned block_mask = (in_block >= 32 ? 0xffffffffu : ((1u << in_block) - 1u));
    if (((showing >> z0) & block_mask) == 0u) {
      if (tid == 0) {
        bulk_store_obs(obs_t + (warp_base + z0) * (int64_t)K, cta_zero, (uint32_t)in_block * (uint32_t)K * (uint32_t)sizeof(O));
        bulk_commit();
      }
      continue;
    }
    for (int g0 = z0; g0 < z0 + in_block; g0 += m) {
      const int in_group = (z0 + in_block - g0) < m ? (z0 + in_block - g0) : m;
      O* dst = obs_t + (warp_base + g0) * (int64_t)K;
      const uint32_t bytes = (uint32_t)in_group * (uint32_t)K * (uint32_t)sizeof(O);
      if (tid == 0) bulk_wait_read<0>();      // the previous staged store has finished reading the buffer
      __syncwarp();
      int img[MAXM];
#pragma unroll
      for (int j = 0; j < MAXM; ++j) img[j] = __shfl_sync(0xffffffffu, image, (g0 + j) & 31);
      for (int q0 = 0; q0 < K16; q0 += 64) {
        uint4 c[MAXM][2];
#pragma unroll
        for (int j = 0; j < MAXM; ++j)
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int q = q0 + r * 32 + tid;
            c[j][r] = make_uint4(0u, 0u, 0u, 0u);
            if (j < in_group && img[j] >= 0 && q < K16)
              c[j][r] = __ldg(reinterpret_cast<const uint4*>(p.images + (int64_t)img[j] * K) + q);
          }
#pragma unroll
        for (int j = 0; j < MAXM; ++j)
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            const int q = q0 + r * 32 + tid;
            if (j < in_group && q < K16) {
              typename Quad<O>::type* out = reinterpret_cast<typename Quad<O>::type*>(buf + (size_t)j * K) + 4 * q;
              out[0] = Quad<O>::of(pixels4(c[j][r].x)); out[1] = Quad<O>::of(pixels4(c[j][r].y));
              out[2] = Quad<O>::of(pixels4(c[j][r].z)); out[3] = Quad<O>::of(pixels4(c[j][r].w));
            }
          }
      }
      fence_proxy_async_smem();
      __syncwarp();
      if (tid == 0) { bulk_store_obs(dst, buf, bytes); bulk_commit(); }
    }
  }
}

// Stream the warp's staged [n_lanes, K] block with ordinary stores (ragged tail warps, unaligned buffers).
// (16-byte moves whatever the element type; the alignment argument of emit_twohot_vec holds for rows too.)
template <class O>
__device__ __forceinline__ void flush_rows_vec(const O* stage, O* obs_t, int64_t warp_base, int n_lanes, int K, bool vec) {
  const int tid = threadIdx.x & 31;
  const int total = n_lanes * K;
  O* dst = obs_t + warp_base * (int64_t)K;
  constexpr int S = Vec16<O>::shift;
  if (vec && (total & ((1 << S) - 1)) == 0) {
    const float4* s4 = reinterpret_cast<const float4*>(stage);
    for (int q = tid; q < (total >> S); q += 32) st_stream(reinterpret_cast<float4*>(dst) + q, s4[q]);
  } else {
    for (int e = tid; e < total; e += 32) st_stream(dst + e, stage[e]);
  }
}

// ----- per-family glue ------------------------------------------------------------
template <class F, class R> struct RowRenderer {
  template <class O> static __device__ __forceinline__ void run(const EnvParams& p, const typename F::Lane& L, R&, O* dst) { F::row(p, L, dst, 1); }
};
template <class R> struct RowRenderer<UmbrellaChain, R> {   // the observation itself draws from the stream
  template <class O> static __device__ __forceinline__ void run(const EnvParams& p, const UmbrellaChain::Lane& L, R& r, O* dst) { UmbrellaChain::row(p, L, r, dst, 1); }
};
template <class R> struct RowRenderer<DeepSea, R> { template <class O> static __device__ __forceinline__ void run(const EnvParams&, const DeepSea::Lane&, R&, O*) {} };
template <class R> struct RowRenderer<Catch, R> { template <class O> static __device__ __forceinline__ void run(const EnvParams&, const Catch::Lane&, R&, O*) {} };
template <class R> struct RowRenderer<Mnist, R> { template <class O> static __device__ __forceinline__ void run(const EnvParams&, const Mnist::Lane&, R&, O*) {} };

template <class F> struct Descriptor {
  static __device__ __forceinline__ int a(const typename F::Lane&) { return -1; }
  static __device__ __forceinline__ int b(const typename F::Lane&) { return -1; }
};
template <> struct Descriptor<DeepSea> {
  static __device__ __forceinline__ int a(const DeepSea::Lane& L) { return L.hot; }
  static __device__ __forceinline__ int b(const DeepSea::Lane&) { return -1; }
};
template <> struct Descriptor<Catch> {
  static __device__ __forceinline__ int a(const Catch::Lane& L) { return L.hot_a; }
  static __device__ __forceinline__ int b(const Catch::Lane& L) { return L.hot_b; }
};
template <> struct Descriptor<Mnist> {
  static __device__ __forceinline__ int a(const Mnist::Lane& L) { return L.image; }
  static __device__ __forceinline__ int b(const Mnist::Lane&) { return -1; }
};

// ----- the fused transition kernel ----------------------------------------------
// Work unit: a CHUNK of 32 consecutive lanes, processed by one warp (thread = lane).  When the batch is too small
// to give every SM a few warps that way and the emitter walks the chunk's lanes serially (mnist images), the host
// shrinks chunks to 16 or 8 lanes (a.chunk_lanes): the transition then idles some threads, which costs nothing
// next to spreading 4 096 lanes x 3 KB over 512 warps instead of 128.
//   * default launch: one chunk per warp, ceil(B / 32) warps; small CTAs (64 threads) keep the per-SM share of
//     the 2048 chunks of a 65 536-lane batch within ~1% of even on 132 SMs and let the hardware CTA scheduler
//     balance SMs dynamically.
//   * deep_sea bulk path: a PERSISTENT grid (as many warps as fit the SMs' shared memory: 3 per SM at N = 32)
//     whose warps pull chunk indices from a global counter (atomicAdd by the elected lane).  SMs drain HBM at
//     slightly different rates (L2 slice / die distance), so dynamic dealing matters -- and so does not reserving
//     work early: LAZY (fetch only after the current chunk's stores are issued; the default).  The TMA unit keeps
//     draining the warp's last two stores while it fetches and loads the next chunk's state.  Every warp's
//     first chunk is its own index (no atomic on the start-up path); the counter deals the rest and is never
//     reset: a launch with C chunks and W warps performs exactly C atomicAdds (C - W successful fetches plus one
//     failing fetch per warp), so launch k starts at work_base_k = work_base_(k-1) + C.
// Graph-safe mode (a.clock != null; the handle switches to it for good the first time one of its launches is
// captured into a CUDA graph): launch arguments are frozen in a graph, so everything that changes from launch to
// launch lives in device memory instead (layout: CLOCK_* below): the steps this handle has advanced since the
// switch (step index = a.step0 + that count: the on-device action stream and the Logging columns depend on it), the
// chunk counter, and the count of finished CTAs.  The CTA that finishes last advances the step count by T and
// zeroes the other two; every CTA reads the step count before it counts itself finished, so the update cannot
// overtake a reader.
// Register budget per family (second __launch_bounds__ argument, counted in 128-thread blocks per SM).  The
// generic kernel is register-hungry (two Philox streams, action stream, accumulators); left alone ptxas takes
// 160-220 registers and 64-thread CTAs then run at 8 warps/SM, which starves the latency-bound small families.
// The caps below double the resident warps of the small families; bandit / discounting_chain go further (<= 64).
template <class F> struct MinBlocksPerSM { static const int value = 4; };        // <= 128 registers
template <> struct MinBlocksPerSM<MemoryChain> { static const int value = 6; };   // <= 80
template <> struct MinBlocksPerSM<Bandit> { static const int value = 8; };        // <= 64
template <> struct MinBlocksPerSM<DiscountingChain> { static const int value = 8; };
#define BSB_LAUNCH_MIN_BLOCKS(V) MinBlocksPerSM<typename V::Fam>::value
// System-scope stores to the pinned mailbox (host memory over PCIe).
__device__ __forceinline__ void st_sys_u64(volatile unsigned long long* ptr, unsigned long long v) {
  asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(ptr), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long global_timer_ns() {
  unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t;
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// Graph-safe mode keeps the step count, the chunk counter and the finished-CTA count in device memory.  Every
// word that many CTAs touch is spread over CLOCK_GROUPS 128-byte lines, because same-line traffic serialises in
// one L2 slice (~2 ns per access): a 16 384-CTA launch reads the step count once per warp and counts itself out
// once per CTA.
//   clock[16 r]                 r < 32: the step count, REPLICATED (CTA b reads replica b % 32; the last CTA of
//                               a launch rewrites all 32); the host reads / writes replica 0 .. 31
//   clock[CLOCK_CHUNK]          chunk counter of the persistent grids (a line of its own)
//   clock[CLOCK_TOP]            groups that have finished
//   clock[CLOCK_SUB0 + 16 g]    CTAs of group g (= blockIdx % 32) that have finished
static const int CLOCK_GROUPS = 32, CLOCK_CHUNK = 16 * CLOCK_GROUPS, CLOCK_TOP = CLOCK_CHUNK + 16,
                 CLOCK_SUB0 = CLOCK_TOP + 16, CLOCK_WORDS = CLOCK_SUB0 + 16 * CLOCK_GROUPS;

// ----- pieces both kernels share ----------------------------------------------------------------------------------
// Per-warp staging state of the observation emitters; it persists across the chunks and steps of a launch.  The
// stages hold observation elements of type O (the mnist table in front of them is float32).
template <class O>
struct WarpStage {
  O* stage;                // this warp's shared-memory stages
  O* cta_zero;             // mnist bulk path: all-zero tiles shared by the CTA's warps (source of the LAST-frame stores)
  unsigned row_mask;       // row / board stage of store number n: n & row_mask
  unsigned emitted = 0;    // bulk stores issued by this warp so far (double-buffer parity)
  int poked_a0 = -1, poked_b0 = -1, poked_a1 = -1, poked_b1 = -1;   // catch: cells poked into stage buffer 0 / 1
  int tile_poked0 = -1, tile_poked1 = -1;      // deep_sea bulk path: cell this thread poked into group buffer 0 / 1
  bool any_bulk = false;   // a chunk went through the TMA unit
};

// Carves the warp's stages out of dynamic shared memory and clears those that rely on staying zero between steps
// (before the dependency wait).  Every thread of the CTA calls it.
template <class F, class O>
__device__ __forceinline__ WarpStage<O> clear_stages(const EnvParams& p, const LaunchArgs& a) {
  extern __shared__ float4 smem_raw[];
  constexpr int kEmit = EmitKind<F>::value;
  const int tid = threadIdx.x & 31, warp = threadIdx.x >> 5, warps_per_cta = blockDim.x >> 5;
  constexpr int S = Vec16<O>::shift;
  const size_t stage_elems = smem_elems_per_warp<F, O>(p.obs_numel, a.emit_bulk != 0, a.emit_reuse != 0, a.group_lanes, a.stage_rows);
  WarpStage<O> ws;
  ws.stage = reinterpret_cast<O*>(smem_raw) + (size_t)warp * stage_elems;
  ws.cta_zero = reinterpret_cast<O*>(smem_raw) + (size_t)warps_per_cta * stage_elems;
  ws.row_mask = a.stage_rows == 2 ? 1u : 0u;
  if (kEmit == EMIT_TWOHOT || (kEmit == EMIT_ONEHOT && a.emit_bulk)) {
    float4* s4 = reinterpret_cast<float4*>(ws.stage);
    const int total4 = (int)(stage_elems >> S);
    for (int q = tid; q < total4; q += 32) s4[q] = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int e = (total4 << S) + tid; e < (int)stage_elems; e += 32) ws.stage[e] = obs_cast<O>(0.f);
    __syncwarp();
  }
  if (kEmit == EMIT_IMAGE) {      // pixel table: image.astype(float32) / 255 for every int8 value (mnist.py:64)
    for (int i = tid; i < 256; i += 32) reinterpret_cast<float*>(ws.stage)[i] = Mnist::pixel((int8_t)(uint8_t)i);
    for (int i = threadIdx.x; i < a.cta_extra_elems; i += blockDim.x) ws.cta_zero[i] = obs_cast<O>(0.f);
    fence_proxy_async_smem();
    __syncthreads();
  }
  return ws;
}

// The elected lane draws chunk indices [total_warps, n_chunks) from the global counter and broadcasts them with a
// shuffle (chunk = global warp index is taken without asking).
__device__ __forceinline__ int64_t fetch_chunk(const LaunchArgs& a, int64_t total_warps) {
  unsigned long long v = 0;
  if ((threadIdx.x & 31) == 0) v = atomicAdd(a.work_counter, 1ull) - a.work_base;      // graph-safe mode: clock + 1, base 0
  return total_warps + (int64_t)__shfl_sync(0xffffffffu, v, 0);
}

// Which chunks leave through the TMA unit (spans that are whole multiples of 16 bytes, from 16-byte aligned starts:
// see emit_twohot_vec); warp-uniform per chunk.
template <class F, class O>
__device__ __forceinline__ bool chunk_is_bulk(const EnvParams& p, const LaunchArgs& a, bool vec, int n_lanes) {
  constexpr int kEmit = EmitKind<F>::value;
  constexpr int V1 = (1 << Vec16<O>::shift) - 1;     // elements per 16 bytes, minus one
  const int K = p.obs_numel;
  bool bulk = a.emit_bulk && vec;
  if (kEmit == EMIT_ROWS) bulk = bulk && K >= 3 && ((n_lanes * K) & V1) == 0;
  if (kEmit == EMIT_TWOHOT) bulk = bulk && ((n_lanes * K) & V1) == 0;
  if (kEmit == EMIT_ONEHOT) bulk = bulk && ((K & V1) == 0 || ((n_lanes % a.group_lanes) == 0 && ((a.group_lanes * K) & V1) == 0));
  if (kEmit == EMIT_IMAGE) bulk = bulk && (K & 3) == 0;
  return bulk;
}
// Whether a one-hot chunk that does not go through the TMA unit goes through emit_onehot_reuse: the launch asks for
// it and the tiles are whole 16-byte words.
template <class O>
__device__ __forceinline__ bool reuse_chunk(const LaunchArgs& a, bool vec, int K) {
  return a.emit_reuse && vec && (K & ((1 << Vec16<O>::shift) - 1)) == 0;
}

// Observation emitter of the warp for one chunk and step.  Every element is converted where it is written to the
// stage or to global memory (obs_cast).  `reuse`: one-hot tiles may go through emit_onehot_reuse (the launch's
// observations; final observations of same-step handles, whose buffer the launch plan did not look at, never do).
template <class F, class O, class R>
__device__ __forceinline__ void emit_obs(const EnvParams& p, const LaunchArgs& a, WarpStage<O>& ws, const typename F::Lane& L,
                                         R& rng, O* obs_t, int64_t warp_base, int n_lanes, int64_t lane, bool active,
                                         bool bulk, bool vec, bool reuse = true) {
  constexpr int kEmit = EmitKind<F>::value;
  constexpr int V1 = (1 << Vec16<O>::shift) - 1;
  const int tid = threadIdx.x & 31;
  const int K = p.obs_numel;
  if (kEmit == EMIT_ONEHOT) {
    const int hot = Descriptor<F>::a(L);
    if (bulk) {
      // Groups of m consecutive lanes share one staging buffer (m tiles, contiguous in global memory too) and
      // leave as ONE bulk store of up to m * 4K bytes: large stores amortise the per-operation cost of the
      // TMA unit.
      const int m = a.group_lanes;
      for (int g0 = 0; g0 < n_lanes; g0 += m) {
        const int in_group = (n_lanes - g0) < m ? (n_lanes - g0) : m;
        const int s = (int)(ws.emitted & 1u);
        O* group = ws.stage + (size_t)s * m * K;
        if (tid == 0) bulk_wait_read<TILE_STAGES - 1>();    // the store two back, last reader of `group`, is done
        __syncwarp();
        if (s == 0) { if (ws.tile_poked0 >= 0) { group[ws.tile_poked0] = obs_cast<O>(0.f); ws.tile_poked0 = -1; } }
        else        { if (ws.tile_poked1 >= 0) { group[ws.tile_poked1] = obs_cast<O>(0.f); ws.tile_poked1 = -1; } }
        __syncwarp();     // a thread of an earlier group may clear the very cell another thread sets now
        if (tid >= g0 && tid < g0 + in_group && hot >= 0) {
          const int cell = (tid - g0) * K + hot;
          group[cell] = obs_cast<O>(1.f);
          if (s == 0) ws.tile_poked0 = cell; else ws.tile_poked1 = cell;
        }
        fence_proxy_async_smem();
        __syncwarp();
        if (tid == 0) {
          O* tile_dst = obs_t + (warp_base + g0) * (int64_t)K;
          const uint32_t tile_bytes = (uint32_t)in_group * (uint32_t)K * (uint32_t)sizeof(O);
          bulk_store_obs(tile_dst, group, tile_bytes);
          bulk_commit();
        }
        ++ws.emitted;
      }
    } else if (reuse && reuse_chunk<O>(a, vec, K)) {
      emit_onehot_reuse(reinterpret_cast<uint4*>(ws.stage), obs_t, warp_base, n_lanes, K, hot);
    } else {
      emit_onehot_vec(obs_t, warp_base, n_lanes, K, hot, vec && (K & V1) == 0);
    }
  } else if (kEmit == EMIT_TWOHOT) {
    const int hot_a = Descriptor<F>::a(L), hot_b = Descriptor<F>::b(L);
    if (bulk) {
      const int buf = (int)(ws.emitted & ws.row_mask);
      O* boards = ws.stage + (size_t)buf * 32 * K;
      if (tid == 0) { if (ws.row_mask) bulk_wait_read<1>(); else bulk_wait_read<0>(); }   // the store that last read `boards` is done with it
      __syncwarp();
      O* mine = boards + tid * K;
      const int old_a = buf ? ws.poked_a1 : ws.poked_a0, old_b = buf ? ws.poked_b1 : ws.poked_b0;
      if (old_a >= 0) mine[old_a] = obs_cast<O>(0.f);
      if (old_b >= 0) mine[old_b] = obs_cast<O>(0.f);
      int new_a = -1, new_b = -1;
      if (active) { mine[hot_a] = obs_cast<O>(1.f); mine[hot_b] = obs_cast<O>(1.f); new_a = hot_a; new_b = hot_b; }
      if (buf) { ws.poked_a1 = new_a; ws.poked_b1 = new_b; } else { ws.poked_a0 = new_a; ws.poked_b0 = new_b; }
      fence_proxy_async_smem();
      __syncwarp();
      if (tid == 0) { bulk_store_obs(obs_t + warp_base * (int64_t)K, boards, (uint32_t)n_lanes * (uint32_t)K * (uint32_t)sizeof(O)); bulk_commit(); }
      ++ws.emitted;
    } else {
      emit_twohot_vec(obs_t, warp_base, n_lanes, K, hot_a, hot_b, vec);
    }
  } else if (kEmit == EMIT_IMAGE) {
    const int image = Descriptor<F>::a(L);
    if (bulk) emit_image_bulk(p, ws.stage, ws.cta_zero, obs_t, warp_base, n_lanes, K, active ? image : -1, a.group_lanes,
                              a.cta_extra_elems / K);
    else emit_image(p, reinterpret_cast<const float*>(ws.stage), obs_t, warp_base, n_lanes, K, image, vec && (K & 3) == 0);
  } else if (!a.stage_rows) {
    // observation rows too long for a shared-memory stage: every thread renders its row in place.  Never taken by
    // bfloat16 rows: a stage of 32 rows of K <= 1 536 elements (umbrella_chain's longest) always fits.
    if (active) RowRenderer<F, R>::run(p, L, rng, obs_t + lane * (int64_t)K);
  } else {
    O* rows = ws.stage + (size_t)(ws.emitted & ws.row_mask) * 32 * K;
    if (bulk) { if (tid == 0) { if (ws.row_mask) bulk_wait_read<1>(); else bulk_wait_read<0>(); } }
    __syncwarp();
    if (active) RowRenderer<F, R>::run(p, L, rng, rows + tid * K);
    if (bulk) {
      fence_proxy_async_smem();
      __syncwarp();
      if (tid == 0) { bulk_store_obs(obs_t + warp_base * (int64_t)K, rows, (uint32_t)n_lanes * (uint32_t)K * (uint32_t)sizeof(O)); bulk_commit(); }
    } else {
      __syncwarp();
      flush_rows_vec(rows, obs_t, warp_base, n_lanes, K, vec);
    }
    ++ws.emitted;
  }
}

// Same-step handles: the final observation of every lane whose step returned LAST, rendered from the lane as it was
// before the merged reset; the rows of other lanes are left untouched.  Lanes step in lock-step and most episodes
// have a fixed length, so usually the whole chunk finishes together: then its rows leave through the observation's
// own emitter (bulk, vector or scalar stores, by the same rules; never compare-then-store).  Otherwise only the finished lanes' rows are
// written, each by the whole warp with streaming stores (rows: by the lane's own thread).
// Rows are the exception to "the same rules": their stages serve bulk and non-bulk emits alike, and a non-bulk emit
// neither waits for the TMA unit's reads of a stage nor keeps the stage parity in step with the committed groups.
// Within a chunk every row emit must therefore take the same path; when the final observation's buffer and the
// observation's (`obs_bulk`: that chunk's decision) would take different ones, the final rows are rendered straight
// to global memory by their own threads.  Tiles, boards and images only stage their bulk stores, so any mix is safe.
template <class F, class O, class R>
__device__ __forceinline__ void emit_final(const EnvParams& p, const LaunchArgs& a, WarpStage<O>& ws, MergedReset<F, R>& m,
                                           O* fin_t, int64_t warp_base, int n_lanes, int64_t lane, bool active, bool vec,
                                           bool obs_bulk) {
  constexpr int kEmit = EmitKind<F>::value;
  const int tid = threadIdx.x & 31;
  const int K = p.obs_numel;
  const unsigned done = __ballot_sync(0xffffffffu, active && m.done);
  if (done == 0u) return;
  const bool bulk = chunk_is_bulk<F, O>(p, a, vec, n_lanes);
  if (done == (n_lanes >= 32 ? 0xffffffffu : ((1u << n_lanes) - 1u)) && (kEmit != EMIT_ROWS || bulk == obs_bulk)) {
    ws.any_bulk = ws.any_bulk || bulk;
    emit_obs<F>(p, a, ws, m.last, m.rng, fin_t, warp_base, n_lanes, lane, active, bulk, vec, /*reuse=*/false);
    return;
  }
  if (kEmit == EMIT_ROWS) {
    if (m.done && active) RowRenderer<F, R>::run(p, m.last, m.rng, fin_t + lane * (int64_t)K);
    return;
  }
  const int da = Descriptor<F>::a(m.last), db = Descriptor<F>::b(m.last);
  for (unsigned rest = done; rest != 0u; rest &= rest - 1u) {
    const int j = __ffs(rest) - 1;
    const int a0 = __shfl_sync(0xffffffffu, da, j), b0 = __shfl_sync(0xffffffffu, db, j);
    O* dst = fin_t + (warp_base + j) * (int64_t)K;
    if (kEmit == EMIT_IMAGE) {        // mnist's LAST frame is the all-zero tile (mnist.py:74)
      const float* lut = reinterpret_cast<const float*>(ws.stage);
      const int8_t* src = p.images + (int64_t)(a0 < 0 ? 0 : a0) * K;
      for (int e = tid; e < K; e += 32) st_stream(dst + e, obs_cast<O>(a0 >= 0 ? lut[(uint8_t)src[e]] : 0.f));
    } else {                          // one-hot (b0 = -1) and two-hot boards
      for (int e = tid; e < K; e += 32) st_stream(dst + e, obs_cast<O>((e == a0 || e == b0) ? 1.f : 0.f));
    }
  }
}

// The warp is done: shared memory must outlive its last bulk read.  `drain`: the stores themselves must have
// completed (a single-phase host step's `done` tells the host that the observations are in device memory).
template <class O>
__device__ __forceinline__ void retire_warp(const LaunchArgs& a, const WarpStage<O>& ws, bool drain) {
  if (ws.any_bulk && (threadIdx.x & 31) == 0) { if (drain) bulk_wait_all(); else bulk_wait_read<0>(); }
  if (a.timing && a.mail && threadIdx.x == 0) atomicMax(&a.mail->last_exit, global_timer_ns());
}

// Completion of a host step: every CTA counts itself finished once its zero-copy outputs are visible to the host;
// the last one stores the ticket into the mailbox.
__device__ __forceinline__ void signal_done(const LaunchArgs& a) {
  __threadfence_system();                  // every thread: its zero-copy outputs are visible to the host ...
  __syncthreads();                         // ... before the CTA counts itself finished
  if (threadIdx.x == 0 && atomicAdd(&a.mail->finished, 1ull) == (unsigned long long)gridDim.x - 1ull) {
    a.mail->finished = 0ull;
    __threadfence_system();
    st_sys_u64(&a.mailbox->done, a.ticket);
  }
}

// The chunk loop of a ragged pack (Variant<F, float, RAGGED>).  Setting k owns ceil(L / chunk_lanes) chunks, the last
// possibly partial, so a chunk never straddles two settings: the setting's parameters (K, N, mapping bits, group
// size) are warp-uniform, looked up once per chunk and kept for all T steps.  Row j of setting k's observation block
// receives lane j of the setting.  Tile groups and row stages sit at offsets that depend on the setting's K, so a
// persistent warp (deep_sea bulk path) that moves on to another setting first waits until the TMA unit has read its
// stages, then clears the cells it poked there with the old geometry: the stage is all zeros again before the new
// setting's first poke.
template <class Fam, class R, bool kNoise, bool kTrack>
__device__ __forceinline__ void ragged_chunks(const EnvParams& p, const LaunchArgs& a, WarpStage<float>& ws, int64_t step0,
                                              const MailFields& out, bool vec) {
  constexpr int kEmit = EmitKind<Fam>::value;
  const int tid = threadIdx.x & 31, warp = threadIdx.x >> 5, warps_per_cta = blockDim.x >> 5;
  const RaggedTable* table = reinterpret_cast<const RaggedTable*>(p.pack);
  const int64_t lanes = table->pack.lanes_per_setting, step_elems = table->step_elems;
  const int cl = a.chunk_lanes;
  const int64_t per_setting = (lanes + cl - 1) / cl;
  const int64_t n_chunks = table->pack.n_settings * per_setting;
  const bool dynamic = a.work_counter != nullptr;
  const int64_t total_warps = (int64_t)gridDim.x * warps_per_cta;
  int64_t cur_chunk = (int64_t)blockIdx.x * warps_per_cta + warp;
  int64_t k_prev = -1;
  EnvParams lp = p;              // setting k_prev's parameters
  LaunchArgs la = a;             // ... its lanes per bulk store
  float* obs_k = a.obs;          // ... and its observation block
  bool tiles_bulk = false;       // ... whose tiles may go through the TMA unit
  int group_stride = 0;          // elements from the stage's first tile group to its second

  while (cur_chunk < n_chunks) {
    const int64_t k = cur_chunk / per_setting;
    const int64_t local_base = (cur_chunk - k * per_setting) * cl;      // first lane of the chunk within its setting
    const int n_lanes = (lanes - local_base) < cl ? (int)(lanes - local_base) : cl;
    const int64_t lane = k * lanes + local_base + tid;                 // the pack's lane: state, scalars, accumulators
    const bool active = tid < n_lanes;
    if (k != k_prev) {
      if (k_prev >= 0 && ws.any_bulk) {
        if (tid == 0) bulk_wait_read<0>();
        __syncwarp();
        if (kEmit == EMIT_ONEHOT) {
          if (ws.tile_poked0 >= 0) ws.stage[ws.tile_poked0] = 0.f;
          if (ws.tile_poked1 >= 0) ws.stage[group_stride + ws.tile_poked1] = 0.f;
          ws.tile_poked0 = ws.tile_poked1 = -1;
          __syncwarp();
        }
      }
      const RaggedSetting& s = ragged_setting(table, k);
      lp = p;
      ragged_setting_params(lp, s, table->mapping_bits);
      la.group_lanes = s.group_lanes > 0 ? s.group_lanes : 1;
      tiles_bulk = s.group_lanes > 0;
      group_stride = la.group_lanes * lp.obs_numel;
      obs_k = a.obs + s.obs_offset;
      k_prev = k;
    }
    const bool bulk = chunk_is_bulk<Fam, float>(lp, la, vec, n_lanes) && (kEmit != EMIT_ONEHOT || tiles_bulk);
    ws.any_bulk = ws.any_bulk || bulk;

    typename Fam::Lane L;
    R rng, wrng;
    EpisodeStats ep;
    ActionStream action_stream;
    action_stream.open();
    if (active) lane_open<Fam>(lp, lane, L, rng, wrng, ep, a.mode, kNoise, kTrack);
    else Fam::init(p, L);
    if (a.mode == MODE_INIT && active) Fam::ctor_draws(lp, L, rng);      // the constructor runs no step (T = 0)

    for (int64_t t = 0; t < a.T; ++t) {
      const int64_t off = t * p.batch + lane;
      if (active) {
        int32_t action = 0;
        if (a.mode == MODE_STEP) {
          if (a.actions) {
            action = a.actions[off];
            if ((uint32_t)action >= (uint32_t)p.num_actions) {
              if (a.bad_action) *a.bad_action = 1;
              action = action < 0 ? 0 : p.num_actions - 1;
            }
          } else {
            action = action_stream.sample(a.action_seed, lp.lane_offset + (uint64_t)lane, (uint64_t)(step0 + t), p.num_actions);
          }
          if (a.actions_out) a.actions_out[off] = action;
        }
        lane_step<Fam>(lp, lane, L, rng, wrng, ep, action, a.mode, kNoise, kTrack, step0 + t, out, off);
      }
      emit_obs<Fam>(lp, la, ws, L, rng, obs_k + t * step_elems, local_base, n_lanes, local_base + tid, active, bulk, vec);
    }

    if (active) lane_close<Fam>(lp, lane, L, rng, wrng, ep, kNoise, kTrack);
    cur_chunk = dynamic ? fetch_chunk(a, total_warps) : n_chunks;
  }
}

// The fused transition kernel: ordinary launches (constructor, reset, step, rollout), graph-safe mode and the
// single-phase host step.
template <class V, int RK, bool kNoise, bool kTrack>
__global__ void __launch_bounds__(128, BSB_LAUNCH_MIN_BLOCKS(V)) transition_kernel(const EnvParams p, const LaunchArgs a) {
  typedef typename V::Fam Fam;
  typedef typename V::Obs O;
  typedef typename RngOf<RK>::type R;
  constexpr bool kSameStep = V::kSameStep;
  constexpr bool kPacked = V::kPacked;
  const int tid = threadIdx.x & 31, warp = threadIdx.x >> 5, warps_per_cta = blockDim.x >> 5;
  const int64_t B = p.batch;
  const int K = p.obs_numel;
  WarpStage<O> ws = clear_stages<Fam, O>(p, a);
  // Wait for the previous step's kernel (it wrote the lane state read below), THEN allow the next step's kernel
  // to become resident: its CTAs park at their own wait, so at most one dependent grid is ever pending.
  if (a.use_pdl) { pdl_wait(); pdl_launch_dependents(); }
  int64_t step0 = a.step0;
  if (a.clock) step0 += (int64_t)*reinterpret_cast<volatile unsigned long long*>(a.clock + 16 * (blockIdx.x % CLOCK_GROUPS));
  const MailFields out = {a.reward, a.reward_f64, a.discount, a.step_type};
  const bool vec = a.obs_vec_ok != 0;
  O* const obs = reinterpret_cast<O*>(a.obs);       // the ABI's float* addresses elements of type O

  if constexpr (V::kRagged) {
    ragged_chunks<Fam, R, kNoise, kTrack>(p, a, ws, step0, out, vec);
  } else {
  const int cl = a.chunk_lanes;
  const int64_t n_chunks = (B + cl - 1) / cl;
  const bool dynamic = a.work_counter != nullptr;
  const int64_t total_warps = (int64_t)gridDim.x * warps_per_cta;
  int64_t cur_chunk = (int64_t)blockIdx.x * warps_per_cta + warp;

  while (cur_chunk < n_chunks) {
    const int64_t warp_base = cur_chunk * cl;
    const int n_lanes = (B - warp_base) < cl ? (int)(B - warp_base) : cl;
    const int64_t lane = warp_base + tid;
    const bool active = tid < n_lanes;
    const bool bulk = chunk_is_bulk<Fam, O>(p, a, vec, n_lanes);
    ws.any_bulk = ws.any_bulk || bulk;
    // The parameters this lane runs with: p itself, or (packed kernels) a copy with its setting's values, which it
    // keeps for all T steps of the launch.
    EnvParams setting_p;
    if constexpr (kPacked) { setting_p = p; if (active) pack_lane_params(setting_p, lane); }
    const EnvParams& lp = kPacked ? setting_p : p;

    typename Fam::Lane L;
    R rng, wrng;
    EpisodeStats ep;
    ActionStream action_stream;
    action_stream.open();
    if (active) lane_open<Fam>(lp, lane, L, rng, wrng, ep, a.mode, kNoise, kTrack);
    else Fam::init(p, L);
    if (a.mode == MODE_INIT && active) Fam::ctor_draws(lp, L, rng);      // the constructor runs no step (T = 0)
    MergedReset<Fam, R> merged;            // same-step kernels only
    if constexpr (kSameStep) { Fam::init(p, merged.last); merged.done = false; }

    for (int64_t t = 0; t < a.T; ++t) {
      const int64_t off = t * B + lane;
      if (active) {
        int32_t action = 0;
        if (a.mode == MODE_STEP) {
          if (a.actions) {
            action = a.actions[off];
            if ((uint32_t)action >= (uint32_t)p.num_actions) {      // never index a table or pack state with it
              if (a.bad_action) *a.bad_action = 1;
              action = action < 0 ? 0 : p.num_actions - 1;
            }
          } else {
            action = action_stream.sample(a.action_seed, lp.lane_offset + (uint64_t)lane, (uint64_t)(step0 + t), p.num_actions);
          }
          if (a.actions_out) a.actions_out[off] = action;
        }
        if constexpr (kSameStep) lane_step<Fam, R, true>(p, lane, L, rng, wrng, ep, action, a.mode, kNoise, kTrack, step0 + t, out, off, &merged);
        else lane_step<Fam>(lp, lane, L, rng, wrng, ep, action, a.mode, kNoise, kTrack, step0 + t, out, off);
      }
      if constexpr (kSameStep) {
        if (a.final_obs)
          emit_final<Fam>(p, a, ws, merged, reinterpret_cast<O*>(a.final_obs) + t * B * (int64_t)K, warp_base, n_lanes,
                          lane, active, a.final_vec_ok != 0, bulk);
      }
      emit_obs<Fam>(lp, a, ws, L, rng, obs + t * B * (int64_t)K, warp_base, n_lanes, lane, active, bulk, vec);
    }

    if (active) lane_close<Fam>(lp, lane, L, rng, wrng, ep, kNoise, kTrack);
    // a persistent warp reserves its next chunk only once this one's stores are issued
    cur_chunk = dynamic ? fetch_chunk(a, total_warps) : n_chunks;
  }
  }  // !V::kRagged
  retire_warp(a, ws, a.mailbox != nullptr);
  if (a.mailbox) signal_done(a);
  if (a.clock) {
    __syncthreads();
    if (threadIdx.x == 0) {
      const unsigned groups = gridDim.x < (unsigned)CLOCK_GROUPS ? gridDim.x : (unsigned)CLOCK_GROUPS;
      const unsigned g = blockIdx.x % groups;
      const unsigned members = gridDim.x / groups + (g < gridDim.x % groups ? 1u : 0u);
      unsigned long long* sub = a.clock + CLOCK_SUB0 + 16 * g;
      // No fence: the count only says "this CTA has READ the step count and drawn its chunks" -- both happened
      // (their values were consumed) long before; the state it wrote reaches the next launch through the kernel
      // boundary.  A membar here kept every CTA alive ~1 us longer: +2..7 us per launch on multi-wave grids.
      if (atomicAdd(sub, 1ull) == (unsigned long long)members - 1ull) {
        *sub = 0ull;                          // re-armed for the next launch (which starts after this one ends)
        if (atomicAdd(a.clock + CLOCK_TOP, 1ull) == (unsigned long long)groups - 1ull) {
          const unsigned long long steps = (unsigned long long)(step0 - a.step0) + (a.mode == MODE_INIT ? 0ull : (unsigned long long)a.T);
          for (int r = 0; r < CLOCK_GROUPS; ++r) a.clock[16 * r] = steps;
          a.clock[CLOCK_CHUNK] = 0ull;
          a.clock[CLOCK_TOP] = 0ull;
        }
      }
    }
  }
}

// ----- the two-phase host step ------------------------------------------------------------------------------------
// Families whose observation is a function of the STORED lane state (ObsFromState: deep_sea, catch), host-driven
// steps (bsb_step_host) on pinned buffers.  Such a step returns when reward / discount / step_type are in host
// memory; the observation stays on the device.  So the transitions of ALL chunks run first (phase 1: statically
// dealt; the actions of a warp's chunks are fetched in one round trip), and the observations are streamed
// afterwards (phase 2, dynamically dealt as usual) while the host already decides the next action.  Phase 2
// re-reads the lane state phase 1 stored (L2-resident) and renders from it; a warp's first chunk stays in
// registers.
// Who ships the scalars to the host?  Not the workers: 768 KB of posted PCIe writes per step back-pressure the
// warps that issue them (tools/e2e_timeline.py shows it: a phase 1 that writes to host memory takes several times
// longer), and they have 268 MB of observations to issue.  The workers write reward / discount / step_type to a
// DEVICE staging block, fence at GPU scope and count themselves out.  The first `h.copiers` blocks, the COPIERS, own
// no chunks at first: they wait for that count, copy the staging block to the host's pinned buffers with 16-byte
// stores (16 per thread in flight: ~128 KB across the copiers, enough for the link), issue the system fence, and
// the last one stores the completion word; then they join phase 2 through the chunk counter like everybody else.
// (PTX memory model: workers release / copiers acquire at gpu scope; the copiers' own stores, fence.sc.sys and the
// completion word are program-ordered; the host's acquire load of the word therefore sees every scalar.)
// Every host step, BSB_HOST_NO_WAIT included, is one launch of this kernel.  Host steps never run in graph-safe
// mode (the launcher checks): there is no device clock here.
template <class V, int RK, bool kNoise, bool kTrack>
__global__ void __launch_bounds__(128, BSB_LAUNCH_MIN_BLOCKS(V))
two_phase_host_kernel(const EnvParams p, const LaunchArgs a, const TwoPhaseArgs h) {
  typedef typename V::Fam Fam;
  typedef typename V::Obs O;
  static_assert(!V::kSameStep && !V::kPacked, "the two-phase host step runs next-step handles");
  static_assert(ObsFromState<Fam>::value, "the two-phase host step renders observations from the stored lane state");
  typedef typename RngOf<RK>::type R;
  const int tid = threadIdx.x & 31, warp = threadIdx.x >> 5, warps_per_cta = blockDim.x >> 5;
  const int64_t B = p.batch;
  WarpStage<O> ws = clear_stages<Fam, O>(p, a);
  if (a.use_pdl) { pdl_wait(); pdl_launch_dependents(); }
  const bool vec = a.obs_vec_ok != 0;
  O* const obs = reinterpret_cast<O*>(a.obs);       // the ABI's float* addresses elements of type O

  const int cl = a.chunk_lanes;
  const int64_t n_chunks = (B + cl - 1) / cl;
  const bool dynamic = a.work_counter != nullptr;
  const unsigned copier_blocks = (unsigned)h.copiers;
  const unsigned worker_blocks = gridDim.x - copier_blocks;
  const int64_t total_warps = (int64_t)worker_blocks * warps_per_cta;
  const int64_t own = (int64_t)(blockIdx.x - copier_blocks) * warps_per_cta + warp;      // workers only

  // Phase 2: streams the observations of chunk c and of every chunk the counter deals after it, rendered from the
  // stored lane state.  `kept`: chunk c is the warp's own, its state `first` still in registers from phase 1.
  auto render_stored = [&](int64_t c, bool kept, const typename Fam::Lane& first) {
    while (c < n_chunks) {
      const int64_t warp_base = c * cl;
      const int n_lanes = (B - warp_base) < cl ? (int)(B - warp_base) : cl;
      const int64_t lane = warp_base + tid;
      const bool active = tid < n_lanes;
      typename Fam::Lane L = first;
      if (!kept) {
        // some other warp ran this chunk's phase 1 -- long ago in practice, but wait for every chunk's
        if (tid == 0) while (a.mail->phase1 != a.ticket) {}
        __syncwarp();
        __threadfence();                   // acquire: the loads below must not be served from a stale L1 line
        Fam::init(p, L);
        if (active) { Fam::load(p, lane, L); Fam::describe(p, L); }
      }
      const bool bulk = chunk_is_bulk<Fam, O>(p, a, vec, n_lanes);
      ws.any_bulk = ws.any_bulk || bulk;
      R unused_rng;
      emit_obs<Fam>(p, a, ws, L, unused_rng, obs, warp_base, n_lanes, lane, active, bulk, vec);
      kept = false;
      c = dynamic ? fetch_chunk(a, total_warps) : n_chunks;
    }
  };
  typename Fam::Lane keep;
  Fam::init(p, keep);

  if (blockIdx.x < copier_blocks) {
    if (threadIdx.x == 0) {
      const unsigned long long t_start = a.timing ? global_timer_ns() : 0ull;
      while (*reinterpret_cast<volatile unsigned long long*>(&a.mail->finished) < (unsigned long long)worker_blocks) {}
      if (blockIdx.x == 0) {
        a.mail->phase1 = a.ticket;         // every chunk's state is stored: phase 2 may read any lane's state
        if (a.timing) {
          st_sys_u64(&a.mailbox->stamp[0], t_start);
          st_sys_u64(&a.mailbox->stamp[1], global_timer_ns());
          st_sys_u64(&a.mailbox->stamp[3], a.mail->last_exit);
        }
      }
    }
    __syncthreads();
    __threadfence();                       // acquire: the staging block is read below
    const int64_t n_thr = (int64_t)copier_blocks * blockDim.x, me = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    auto ship = [&](const void* from, void* to, int64_t bytes) {
      if (!from || !to) return;
      if ((reinterpret_cast<uintptr_t>(from) | reinterpret_cast<uintptr_t>(to)) & 15) {      // odd batch sizes: words
        const uint32_t* s32 = reinterpret_cast<const uint32_t*>(from);
        uint32_t* d32 = reinterpret_cast<uint32_t*>(to);
        for (int64_t i = me; i < (bytes >> 2); i += n_thr) d32[i] = __ldcg(s32 + i);
        return;
      }
      const uint4* src = reinterpret_cast<const uint4*>(from);
      uint4* dst = reinterpret_cast<uint4*>(to);
      const int64_t n16 = bytes >> 4;
      constexpr int U = 16;     // 16 x 16 B per thread in flight: ~128 KB across the copiers, enough for the PCIe link
      for (int64_t i0 = me; i0 < n16; i0 += U * n_thr) {
        uint4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) { const int64_t i = i0 + u * n_thr; if (i < n16) v[u] = __ldcg(src + i); }
#pragma unroll
        for (int u = 0; u < U; ++u) { const int64_t i = i0 + u * n_thr; if (i < n16) dst[i] = v[u]; }
      }
      const char* tail_src = reinterpret_cast<const char*>(from) + (n16 << 4);
      char* tail_dst = reinterpret_cast<char*>(to) + (n16 << 4);
      for (int64_t i = me; i < (bytes & 15); i += n_thr) tail_dst[i] = tail_src[i];
    };
    ship(h.stage.reward, a.reward, B * 4);
    ship(h.stage.reward_f64, a.reward_f64, B * 8);
    ship(h.stage.discount, a.discount, B * 4);
    ship(h.stage.step_type, a.step_type, B * 4);
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0 && atomicAdd(&a.mail->copied, 1ull) == (unsigned long long)copier_blocks - 1ull) {
      a.mail->finished = 0ull;             // every copier is past its wait: re-arm both counts for the next launch
      a.mail->copied = 0ull;
      __threadfence_system();
      if (a.timing) st_sys_u64(&a.mailbox->stamp[2], global_timer_ns());
      st_sys_u64(&a.mailbox->done, a.ticket);      // the host may read its scalars
    }
    // join phase 2: the copiers own no chunk of their own, the counter deals them the rest
    render_stored(dynamic ? fetch_chunk(a, total_warps) : n_chunks, false, keep);
  } else {
    constexpr int kAhead = 4;              // chunks whose loads (action, lane state, accumulators) are in flight together
    for (int64_t c0 = own; c0 < n_chunks; c0 += kAhead * total_warps) {
      // every independent load of up to kAhead chunks first: one round trip to L2 instead of one per chunk -- a warp
      // owns 4-5 chunks of a 65 536-lane batch
      int32_t fetched[kAhead];
      typename Fam::Lane lanes[kAhead];
      EpisodeStats eps[kAhead];
#pragma unroll
      for (int k = 0; k < kAhead; ++k) {
        const int64_t c = c0 + k * total_warps;
        const int64_t lane = c * cl + tid;
        const bool live = c < n_chunks && tid < cl && lane < B;
        fetched[k] = 0;
        Fam::init(p, lanes[k]);
        if (live) {
          fetched[k] = a.actions[lane];
          Fam::load(p, lane, lanes[k]);
          if (kTrack) eps[k].load(p, lane);
        }
      }
#pragma unroll
      for (int k = 0; k < kAhead; ++k) {
        const int64_t c = c0 + k * total_warps;
        if (c >= n_chunks) break;
        const int64_t lane = c * cl + tid;
        typename Fam::Lane& L = lanes[k];
        if (tid < cl && lane < B) {
          R rng, wrng;
          lane_open<Fam>(p, lane, L, rng, wrng, eps[k], MODE_STEP, kNoise, kTrack, /*state_loaded=*/true);
          int32_t action = fetched[k];
          if ((uint32_t)action >= (uint32_t)p.num_actions) {
            if (a.bad_action) *a.bad_action = 1;
            action = action < 0 ? 0 : p.num_actions - 1;
          }
          lane_step<Fam>(p, lane, L, rng, wrng, eps[k], action, MODE_STEP, kNoise, kTrack, a.step0, h.stage, lane);
          lane_close<Fam>(p, lane, L, rng, wrng, eps[k], kNoise, kTrack);
        }
        if (c == own) keep = L;
      }
    }
    __threadfence();                       // gpu scope (device memory only): the copiers do the system-scope one
    __syncthreads();
    if (threadIdx.x == 0) atomicAdd(&a.mail->finished, 1ull);
    render_stored(own, true, keep);
  }
  retire_warp(a, ws, false);
}

// ----- masked calls -----------------------------------------------------------------------------------------------
// bsb_step_masked / bsb_reset_masked: one call in which lane i acts only where mask[i] != 0.  An active lane makes the
// call an unmasked reset / step would make; an inactive lane makes none (lane_sit_out_calls) and none of its output
// entries is written.  Noise and Logging are runtime flags here (lane_open / lane_step take them as arguments), so
// each variant compiles one masked kernel per bit source.
struct MaskArgs {
  const uint8_t* mask;      // [B], device memory (host steps: pinned host memory's device alias, or device staging)
  int32_t noise, track;     // the RewardNoise stream is live / the Logging accumulators are tracked
  int64_t* episodes_left;   // masked rollouts and host steps: [B] episode budgets, counted down at each LAST (nullable)
  uint8_t* mask_out;        // host steps with budgets: mask[i] is cleared here once lane i's budget is spent;
                            // budgeted steps: the mask itself, cleared for lanes whose budget was spent before the
                            // call (null for every other call)
  // bsb_step_budgeted: the `previous` outputs, which receive the masked-in lanes' current entries of the launch's
  // outputs before the step (null for every other call); prev_vec_ok / prev_final_vec_ok: both observation (final
  // observation) buffers start 16-byte aligned
  float* prev_obs;
  float* prev_reward;
  double* prev_reward_f64;
  float* prev_discount;
  int32_t* prev_step_type;
  float* prev_final_obs;
  int32_t prev_vec_ok, prev_final_vec_ok;
  // bsb_step_budgeted_policy: the agent's values [B, num_actions] (action values or logits), the selection rule
  // (POLICY_*), epsilon and the policy stream's seed (null / 0 for every other call)
  const float* policy_values;
  double policy_epsilon;
  uint64_t policy_seed;
  int32_t policy_kind;
};

// The arguments of a CALL_RECORD launch: MaskArgs grown at its end by the lanes' rings (bsb_replay).  The growth is a
// struct of its own, passed to masked_record_kernel only: a larger MaskArgs changed the code ptxas emits for existing
// masked kernels.  The action source is policy_values when non-null, else a.actions.  rec_vec_ok: both ring
// observation buffers start 16-byte aligned and a slot is a whole number of 16-byte words.
struct RecordArgs : MaskArgs {
  int64_t rec_capacity;
  int64_t* rec_num_added;
  float* rec_obs_tm1;
  int32_t* rec_action;
  float* rec_obs;
  float* rec_reward;
  double* rec_reward_f64;
  float* rec_discount;
  int32_t* rec_step_type;
  int32_t rec_vec_ok;
};

// The arguments of a CALL_SEQUENCE launch: MaskArgs grown at its end by the lanes' sequence buffers (bsb_sequence),
// passed to masked_sequence_kernel only, for the reason RecordArgs is.  The action source is RecordArgs's.
// seq_vec_ok: the observation buffer starts 16-byte aligned and a slot is a whole number of 16-byte words.
struct SequenceArgs : MaskArgs {
  int64_t seq_max_length;
  int64_t* seq_length;
  uint8_t* seq_ready;
  float* seq_obs;
  int32_t* seq_action;
  float* seq_reward;
  double* seq_reward_f64;
  float* seq_discount;
  int32_t* seq_step_type;
  int32_t seq_vec_ok;
};

// The arguments of a CALL_ENSEMBLE launch: RecordArgs grown at its end by boot_dqn's ensemble (bsb_ensemble_policy),
// passed to masked_ensemble_kernel only, for the reason RecordArgs is.  policy_values holds every head's values
// [K, B, num_actions]; the ring fields are null when the step records nothing (rec_num_added decides, at run time).
struct EnsembleArgs : RecordArgs {
  int32_t* ens_heads;
  int32_t ens_num_heads;
};

// What one masked_kernel instantiation runs.  CALL_ROLLOUT: bsb_rollout_masked (T steps, sampled or given actions,
// budgets, actions_out).  CALL_ONE: a masked reset or step (T = 1, the caller's actions, no budgets).  CALL_HOST:
// bsb_step_host_masked (T = 1, the caller's actions, optional budgets, the mask write-back, the mailbox signal).
// CALL_ADVANCE: bsb_advance_masked (T steps of sampled actions, optional budgets, no per-step output at all).
// CALL_BUDGETED: bsb_step_budgeted (CALL_HOST without the mailbox: T = 1, the caller's actions, budgets, the masked-in
// lanes' outputs copied to `previous` first, and the mask cleared for lanes whose budget was spent before the call).
// CALL_POLICY: bsb_step_budgeted_policy (CALL_BUDGETED with each stepping lane's action chosen from its row of the
// policy's values by select_action, and written to actions_out).  CALL_RECORD: bsb_step_budgeted_record
// (CALL_BUDGETED or CALL_POLICY, chosen at run time by m.policy_values, with each transition appended to its lane's
// ring).  CALL_SEQUENCE: bsb_step_budgeted_sequence (CALL_RECORD's step, with each transition appended to its lane's
// sequence buffer instead of a ring).  CALL_ENSEMBLE: bsb_step_budgeted_ensemble (CALL_RECORD's policy step reading
// the row of the lane's active head, the ring write when a replay is given, then the head redrawn at a LAST).
enum CallKind { CALL_ROLLOUT = 0, CALL_ONE = 1, CALL_HOST = 2, CALL_ADVANCE = 3, CALL_BUDGETED = 4, CALL_POLICY = 5,
                CALL_RECORD = 6, CALL_SEQUENCE = 7, CALL_ENSEMBLE = 8 };

// Writes lane j's observation `val(e)` (element e of K) with the whole warp: 16-byte streaming stores when `vec`
// (the row starts 16-byte aligned and is a whole number of 16-byte words), else one element per store.
template <class O, class Val>
__device__ __forceinline__ void store_lane_obs(O* dst, int K, bool vec, const Val& val) {
  constexpr int E = 16 / (int)sizeof(O);
  const int tid = threadIdx.x & 31;
  if (vec) {
    for (int q = tid; q < K / E; q += 32) {
      union { uint4 v; O o[E]; } w;
#pragma unroll
      for (int k = 0; k < E; ++k) w.o[k] = obs_cast<O>(val(q * E + k));
      __stcs(reinterpret_cast<uint4*>(dst) + q, w.v);
    }
  } else {
    for (int e = tid; e < K; e += 32) st_stream(dst + e, obs_cast<O>(val(e)));
  }
}

// The observations of the warp's lanes for which `on` holds, into rows row0 + tid of `block` ([rows, K] elements of
// O); the other rows are not touched.  Rows: each lane's thread renders its own row.  Tiles, boards and images: the
// warp walks the lanes __ballot_sync selects and writes each one.  No TMA bulk store: a whole block would overwrite
// the rows of inactive lanes.
template <class F, class O, class R>
__device__ __forceinline__ void emit_lane_subset(const EnvParams& lp, const typename F::Lane& L, R& rng, O* block, int K,
                                                 int64_t row0, bool on, bool vec_base) {
  constexpr int kEmit = EmitKind<F>::value;
  const int tid = threadIdx.x & 31;
  if (kEmit == EMIT_ROWS) {
    if (on) RowRenderer<F, R>::run(lp, L, rng, block + (row0 + tid) * (int64_t)K);
    return;
  }
  const bool vec = vec_base && ((int64_t)K * (int64_t)sizeof(O)) % 16 == 0;
  const int da = Descriptor<F>::a(L), db = Descriptor<F>::b(L);
  for (unsigned rest = __ballot_sync(0xffffffffu, on); rest != 0u; rest &= rest - 1u) {
    const int j = __ffs(rest) - 1;
    const int a0 = __shfl_sync(0xffffffffu, da, j), b0 = __shfl_sync(0xffffffffu, db, j);
    O* dst = block + (row0 + j) * (int64_t)K;
    if (kEmit == EMIT_IMAGE) {                 // a0 < 0: mnist's all-zero LAST frame (mnist.py:74)
      const int8_t* src = lp.images + (int64_t)(a0 < 0 ? 0 : a0) * K;
      store_lane_obs(dst, K, vec, [&](int e) { return a0 >= 0 ? Mnist::pixel(src[e]) : 0.f; });
    } else {                                   // one-hot tiles (b0 = -1) and two-hot boards
      store_lane_obs(dst, K, vec, [&](int e) { return (e == a0 || e == b0) ? 1.f : 0.f; });
    }
  }
}

// Copies the rows row0 + tid of `src` to `dst` ([rows, K] elements of O, as raw bytes: no cast) for the warp's lanes
// for which `on` holds; the other rows are not touched.  Rows: each lane's thread copies its own row.  Tiles, boards
// and images: the warp walks the lanes __ballot_sync selects and copies each row, with 16-byte loads and stores when
// `vec_base` (both buffers start 16-byte aligned) and the row is a whole number of 16-byte words, as emit_lane_subset
// writes it.
template <class F, class O>
__device__ __forceinline__ void copy_lane_subset(const O* src, O* dst, int K, int64_t row0, bool on, bool vec_base) {
  const int tid = threadIdx.x & 31;
  if (EmitKind<F>::value == EMIT_ROWS) {
    if (on) {
      const O* s = src + (row0 + tid) * (int64_t)K;
      O* d = dst + (row0 + tid) * (int64_t)K;
      for (int e = 0; e < K; ++e) d[e] = s[e];
    }
    return;
  }
  const bool vec = vec_base && ((int64_t)K * (int64_t)sizeof(O)) % 16 == 0;
  for (unsigned rest = __ballot_sync(0xffffffffu, on); rest != 0u; rest &= rest - 1u) {
    const int j = __ffs(rest) - 1;
    const O* s = src + (row0 + j) * (int64_t)K;
    O* d = dst + (row0 + j) * (int64_t)K;
    if (vec) {
      const int words = (int)(((int64_t)K * (int64_t)sizeof(O)) >> 4);
      for (int q = tid; q < words; q += 32) __stcs(reinterpret_cast<uint4*>(d) + q, reinterpret_cast<const uint4*>(s)[q]);
    } else {
      for (int e = tid; e < K; e += 32) d[e] = s[e];
    }
  }
}

// Copies the rows row0 + tid of `src` ([rows, K] elements of O, raw bytes) into the same rows of slot `slot` of `ring`
// (a slot is `stride` elements; `slot` is each lane's own) for the warp's lanes for which `on` holds, with streaming
// stores: copy_lane_subset's walk, with each lane's slot taken from its thread.  `vec_base`: both buffers, and every
// slot of `ring`, start 16-byte aligned.
template <class F, class O>
__device__ __forceinline__ void record_lane_rows(const O* src, O* ring, int64_t stride, int64_t slot, int K, int64_t row0,
                                                 bool on, bool vec_base) {
  const int tid = threadIdx.x & 31;
  if (EmitKind<F>::value == EMIT_ROWS) {
    if (on) {
      const O* s = src + (row0 + tid) * (int64_t)K;
      O* d = ring + slot * stride + (row0 + tid) * (int64_t)K;
      for (int e = 0; e < K; ++e) st_stream(d + e, s[e]);
    }
    return;
  }
  const bool vec = vec_base && ((int64_t)K * (int64_t)sizeof(O)) % 16 == 0;
  for (unsigned rest = __ballot_sync(0xffffffffu, on); rest != 0u; rest &= rest - 1u) {
    const int j = __ffs(rest) - 1;
    const int64_t c = __shfl_sync(0xffffffffu, (long long)slot, j);
    const O* s = src + (row0 + j) * (int64_t)K;
    O* d = ring + c * stride + (row0 + j) * (int64_t)K;
    if (vec) {
      const int words = (int)(((int64_t)K * (int64_t)sizeof(O)) >> 4);
      for (int q = tid; q < words; q += 32) __stcs(reinterpret_cast<uint4*>(d) + q, reinterpret_cast<const uint4*>(s)[q]);
    } else {
      for (int e = tid; e < K; e += 32) st_stream(d + e, s[e]);
    }
  }
}

// Every masked call: a masked reset or step (T = 1, no budgets) or bsb_rollout_masked's T masked steps, in one launch.
// One chunk of 32 lanes per warp; a ragged pack's chunks never straddle two settings, and row j of setting k goes to
// the setting's block (emit_lane_subset).  Lane i is active at step t while mask[i] != 0 and its budget
// (m.episodes_left, when given) is positive; each LAST of an active step takes one from the budget.  So a lane's
// active steps are a prefix of the launch: its state, RNG streams, accumulators and budget stay in registers over
// them, and the calls it sits out all come after its last active one (lane_sit_out_calls, once, after lane_close).  A
// warp whose lanes are all inactive stops stepping.  Graph-safe mode reads the call index from the device clock and
// advances it by T, as transition_kernel does; the mask and the budgets are read (and the budgets written) at every
// launch, so a graph replays with whatever the mask buffer holds and keeps counting the budgets down.  kCall ==
// CALL_ONE: a masked reset or step (T = 1, the caller's actions, no budgets, no actions_out), for which the T loop,
// the action stream and the budget compile out; with them live, masked steps of catch and cartpole took 11-21 %
// longer.  kCall == CALL_HOST: a masked host step, CALL_ONE with the budgets kept, mask[i] cleared in m.mask_out for
// a budgeted lane whose budget is spent after the step, and completion signalled through the mailbox when the launch
// carries one.  No store here is a bulk store, so once every thread has fenced (signal_done) the observations are
// written too: a masked host step is always single-phase.  kCall == CALL_ADVANCE: CALL_ROLLOUT with sampled actions
// and every per-step output compiled out (observations, final observations, scalars, actions_out); where an
// observation would be rendered the lane makes the draws rendering makes (ObsDraws::skip), so its streams end where
// CALL_ROLLOUT's do.  A same-step final observation is rendered from a copy of the stream and is simply not rendered.
// kCall == CALL_BUDGETED: CALL_HOST without the mailbox, where every masked-in lane (budget left or not) first copies
// its current entries of the outputs -- observation row, scalars, final observation -- to `previous`
// (copy_lane_subset; the warp syncs before any new row is written), and a masked-in lane whose budget was spent before
// the call clears its mask byte instead of stepping.  kCall == CALL_POLICY: CALL_BUDGETED where a stepping lane reads
// its row of m.policy_values instead of an action and picks with select_action, keyed by (m.policy_seed, global lane)
// at the call's step index; the pick goes to a.actions_out (nullable) and an invalid row raises a.bad_action.
// kCall == CALL_RECORD: CALL_POLICY when m.policy_values is set, else CALL_BUDGETED; after the step every lane that
// stepped and whose new step type is not FIRST appends (o_tm1, a_tm1, r_t, d_t, o_t) to slot num_added % capacity of
// its ring and counts it.  The rows are copied, never rendered again (rendering draws for some families): o_tm1 from
// the row the lane copied to `previous`, o_t from the row the warp has just emitted (a same-step LAST: the final
// observation), after a __syncwarp.  kCall == CALL_SEQUENCE: CALL_RECORD's step, after which every such lane appends
// (a_tm1, r_t, d_t, o_t) at entry t of its sequence buffer, and o_tm1 at observation slot 0 when t == 0 (a new
// sequence): t is the lane's length, or 0 when the length reached max_length or the entry before it is a LAST (the
// sequence was closed by an earlier call).  Every lane writes its ready flag: set where the append closed the sequence.
// kCall == CALL_ENSEMBLE: CALL_RECORD with a policy, where a stepping lane reads head h = ens_heads[lane] (clamped
// into [0, K) with the invalid-action flag raised when outside it) and selects epsilon-greedily from row (h, lane) of
// policy_values [K, B, num_actions]; the ring write runs when rec_num_added is set; then a lane that stepped and whose
// step ended an episode (the LAST that counts its budget down) writes a new head drawn by ensemble_head at the call's
// step index.  The body (bsb_masked_body.inc) is shared with masked_record_kernel, masked_sequence_kernel and
// masked_ensemble_kernel, which run CALL_RECORD, CALL_SEQUENCE and CALL_ENSEMBLE.
template <class V, int RK, int kCall>
__global__ void __launch_bounds__(128, BSB_LAUNCH_MIN_BLOCKS(V)) masked_kernel(const EnvParams p, const LaunchArgs a, const MaskArgs m) {
#include "bsb_masked_body.inc"
}

// CALL_RECORD: masked_kernel's body with RecordArgs.
template <class V, int RK>
__global__ void __launch_bounds__(128, BSB_LAUNCH_MIN_BLOCKS(V)) masked_record_kernel(const EnvParams p, const LaunchArgs a, const RecordArgs m) {
  constexpr int kCall = CALL_RECORD;
#include "bsb_masked_body.inc"
}

// CALL_SEQUENCE: masked_kernel's body with SequenceArgs.
template <class V, int RK>
__global__ void __launch_bounds__(128, BSB_LAUNCH_MIN_BLOCKS(V)) masked_sequence_kernel(const EnvParams p, const LaunchArgs a, const SequenceArgs m) {
  constexpr int kCall = CALL_SEQUENCE;
#include "bsb_masked_body.inc"
}

// CALL_ENSEMBLE: masked_kernel's body with EnsembleArgs.
template <class V, int RK>
__global__ void __launch_bounds__(128, BSB_LAUNCH_MIN_BLOCKS(V)) masked_ensemble_kernel(const EnvParams p, const LaunchArgs a, const EnsembleArgs m) {
  constexpr int kCall = CALL_ENSEMBLE;
#include "bsb_masked_body.inc"
}

#endif  // __CUDACC__

}  // namespace bsb
