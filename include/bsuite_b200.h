/*
 * bsuite_b200 -- C ABI of the batched bsuite environment engine (sm_90a, H100).
 *
 * This header is the drop-in boundary for the one hot path this repo builds:
 * the per-environment step()/reset() dynamics of google-deepmind/bsuite
 * (reference: bsuite/environments/<name>.py, experiments/cartpole_swingup,
 * utils/wrappers.py::RewardNoise/RewardScale), executed for B independent
 * environment "lanes" in lock-step.
 *
 * The reference has no FFI layer (SURVEY.md 8b): its boundary is the Python
 * object contract of bsuite/environments/base.py:34-77.  Each entry point
 * below names the reference interface it replaces.  The Python binding a
 * maintainer would add is a ctypes stub (INTEGRATION.md); ours lives in
 * bsuite_b200/_lib.py.
 *
 * Conventions
 *   - plain C, no C++/torch types; every function returns a bsb_status.
 *   - buffers are CALLER-OWNED.  For a device environment every pointer in
 *     bsb_outputs / `actions` is a device pointer on that device and the work
 *     is enqueued on `stream` (a cudaStream_t passed as void*; NULL = legacy
 *     default stream).  For a host environment (device == BSB_DEVICE_HOST) the
 *     pointers are host pointers and the call is synchronous.
 *   - the library owns only lane state, RNG counters and config tables.
 *   - calls on one handle are not thread-safe; distinct handles are independent.
 *   - a lane whose previous timestep was LAST ignores its action and emits
 *     FIRST (base.py:59-65), unless the handle was created with
 *     BSB_FLAG_SAME_STEP_RESET (see there).  FIRST lanes carry reward = 0, discount = 0; the
 *     reference's `None` is recovered from step_type == BSB_FIRST.
 */
#ifndef BSUITE_B200_H_
#define BSUITE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BSB_ABI_VERSION 15
#define BSB_DEVICE_HOST (-1)
#define BSB_MAX_INFO 4
#define BSB_MAX_PACKED_SETTINGS 64 /* bsb_create_packed: settings per handle */

typedef enum bsb_status {
  BSB_OK = 0,
  BSB_INVALID_ARGUMENT = 1,
  BSB_UNSUPPORTED = 2,
  BSB_CUDA_ERROR = 3,
  BSB_OUT_OF_MEMORY = 4,
  BSB_INTERNAL = 5
} bsb_status;

/* dm_env.StepType values (dm_env is the reference's L0 substrate). */
typedef enum bsb_step_type { BSB_FIRST = 0, BSB_MID = 1, BSB_LAST = 2 } bsb_step_type;

/* One entry per environment CLASS of the reference (SURVEY.md 8a a2..a11). */
typedef enum bsb_family {
  BSB_DEEP_SEA = 0,          /* environments/deep_sea.py:51-155            */
  BSB_CATCH = 1,             /* environments/catch.py:45-117               */
  BSB_CARTPOLE = 2,          /* environments/cartpole.py:37-181            */
  BSB_CARTPOLE_SWINGUP = 3,  /* experiments/cartpole_swingup/cartpole_swingup.py:41-155 */
  BSB_MOUNTAIN_CAR = 4,      /* environments/mountain_car.py:33-102        */
  BSB_MEMORY_CHAIN = 5,      /* environments/memory_chain.py:37-112        */
  BSB_BANDIT = 6,            /* environments/bandit.py:35-73               */
  BSB_UMBRELLA_CHAIN = 7,    /* environments/umbrella_chain.py:39-114      */
  BSB_DISCOUNTING_CHAIN = 8, /* environments/discounting_chain.py:40-105   */
  BSB_MNIST = 9,             /* environments/mnist.py:36-85                */
  BSB_NUM_FAMILIES = 10
} bsb_family;

/* utils/wrappers.py:250-373, fused into the transition kernel's epilogue. */
typedef enum bsb_wrapper {
  BSB_WRAP_NONE = 0,
  BSB_WRAP_REWARD_NOISE = 1, /* r + noise_scale * randn()   (wrappers.py:275-283) */
  BSB_WRAP_REWARD_SCALE = 2  /* r * reward_scale            (wrappers.py:338-346) */
} bsb_wrapper;

/* Which bit source feeds numpy's legacy RandomState algorithms per lane. */
typedef enum bsb_rng_kind {
  /* Philox4x64-10 (numpy.random.Philox layout): lane i of the batch consumes
   * exactly the stream of numpy.random.RandomState(numpy.random.Philox(
   * key=[seed, lane_offset+i])); the reward wrapper's private RandomState
   * (wrappers.py:267,330) is the same key with counter=[0,0,0,1].           */
  BSB_RNG_PHILOX = 0,
  /* MT19937 exactly as numpy.random.RandomState(seed + lane_offset + i): a
   * B=1 environment then reproduces the UNPATCHED reference for integer
   * seeds.  2.5 KB of generator state per lane; meant for small batches.    */
  BSB_RNG_MT19937 = 1
} bsb_rng_kind;

/*
 * Element type of the observations a handle writes (bsb_config.obs_dtype),
 * fixed at bsb_create.  What is written is exactly the float32 observation
 * converted: bfloat16 rounds to nearest even (as torch.Tensor.to(bfloat16)
 * does; a NaN, which no observation holds, is written as 0x7fc0), uint8
 * holds the 0 / 1 cells of deep_sea and catch.  Reduced dtypes
 * need BSB_RNG_PHILOX; uint8 is for deep_sea and catch only (other
 * combinations return BSB_UNSUPPORTED).  Rewards, discounts, step types, info,
 * episode statistics, log rows and the state snapshot do not depend on it.
 */
typedef enum bsb_obs_dtype {
  BSB_OBS_FLOAT32 = 0,
  BSB_OBS_BFLOAT16 = 1,
  BSB_OBS_UINT8 = 2
} bsb_obs_dtype;

/*
 * Environment configuration: the keyword arguments of the reference
 * constructors, flattened into one POD.  Fields that do not apply to `family`
 * are ignored.  Tables are HOST pointers; bsb_create copies them.
 */
typedef struct bsb_config {
  int32_t family;        /* bsb_family */
  int32_t wrapper;       /* bsb_wrapper */
  int32_t rng_kind;      /* bsb_rng_kind */
  int32_t flags;         /* BSB_FLAG_* */

  /* deep_sea.py:51-57 */
  int32_t size;          /* N */
  int32_t deterministic; /* 1 = deterministic (default), 0 = 'windy' */
  /* catch.py:45-48 */
  int32_t rows, columns;
  /* memory_chain.py:37-40 */
  int32_t memory_length, num_bits;
  /* umbrella_chain.py:39-42 */
  int32_t chain_length, n_distractor;
  /* bandit.py:35 */
  int32_t num_actions;
  /* mountain_car.py:36-38 */
  int32_t max_steps;
  /* mnist.py:36 (num_data = int(fraction * len(labels)), 28x28 images) */
  int32_t num_data, image_rows, image_cols;
  int32_t obs_dtype;     /* bsb_obs_dtype; 0 = float32 */

  double unscaled_move_cost;                         /* deep_sea.py:54 */
  double height_threshold, x_threshold, timescale,   /* cartpole.py:82-87 */
         max_time, init_range;
  double theta_dot_threshold, x_reward_threshold,    /* cartpole_swingup.py:51-60 */
         move_cost;
  double noise_scale;                                /* wrappers.py:253-256 */
  double reward_scale;                               /* wrappers.py:316-319 */

  /* Host tables, built by the caller with the SAME numpy calls the reference
   * constructors make, so they are equal by construction:
   *   deep_sea : uint8  [N*N]  action mapping  (deep_sea.py:79-85)
   *   bandit   : double [num_actions] rewards  (bandit.py:45-47)
   *   discounting_chain : double [5] rewards   (discounting_chain.py:55-56)
   *   mnist    : int8   [num_data*rows*cols] images (utils/datasets.py:52-56) */
  const void* table;
  int64_t table_bytes;
  /*   mnist    : uint8  [num_data] labels */
  const void* table2;
  int64_t table2_bytes;

  /* Log schedule of the reference's Logging wrapper (utils/wrappers.py:99-110,
   * 140-147): the ascending episode counts {1, 1.2, ..., 10} x 10^k up to
   * bsuite_num_episodes at which it writes a row.  When given (host int64
   * array; needs BSB_FLAG_TRACK_EPISODES) every lane records its own row --
   * the five Logging columns + bsuite_info() at that LAST timestep -- on the
   * device (bsb_read_log_rows).  NULL / 0: no rows are recorded. */
  const int64_t* log_schedule;
  int64_t log_schedule_len;
} bsb_config;

/* bsb_config.flags */
#define BSB_FLAG_TRACK_EPISODES 1u /* keep the Logging-wrapper accumulators
                                      (wrappers.py:85-110) per lane on device */
/*
 * Same-step auto-reset, fixed at bsb_create (needs BSB_RNG_PHILOX; MT19937
 * returns BSB_UNSUPPORTED).  A lane whose step returns LAST runs reset() in
 * the SAME call: that call returns LAST with the transition's reward and
 * discount, but its observation is the next episode's FIRST observation, and
 * the lane's next call is an ordinary step.  FIRST is then only returned by
 * the first call of a fresh handle and by bsb_reset.  Per lane this is the
 * reference's own call sequence with every LAST merged into the reset call
 * that follows it: the random draws happen in the reference's order (the
 * step's, the LAST observation's, the reset's, the FIRST observation's), so
 * every value the reference produces appears exactly once.  The observation
 * the reference returned with the LAST goes to bsb_outputs.final_observation
 * when that is given.  Log rows, bsuite_info() and the Logging columns equal
 * the reference's on that folded trace (episode_len / episode_return keep the
 * finished episode's values until the lane steps again).  The snapshot of a
 * same-step handle that tracks episodes holds one more float64 [B] block.
 * Without the flag, behaviour is exactly the default next-step convention.
 */
#define BSB_FLAG_SAME_STEP_RESET 2u

/*
 * Caller-allocated outputs of one lock-step transition.  For bsb_rollout each
 * array carries a leading T axis.  Any pointer except `observation` may be
 * NULL (that output is then not written).
 *   observation : float32 [B, obs_numel]   fresh dense tensor every step
 *                 (a handle created with a reduced obs_dtype writes obs_numel
 *                 elements of THAT type per lane here: the pointer keeps its
 *                 declared type and the caller casts, e.g. (float*)bf16_buffer;
 *                 the same holds for bsb_step_host's device_obs and
 *                 host_out->observation)
 *   reward      : float32 [B]   (float32 rounding of the float64 reward)
 *   reward_f64  : float64 [B]   (the reference's double-precision reward)
 *   discount    : float32 [B]   1 (MID) / 0 (LAST) / 0 (FIRST = None)
 *   step_type   : int32   [B]   bsb_step_type
 *   final_observation : [B, obs_numel] in the handle's obs_dtype, or NULL.
 *                 Same-step handles only (BSB_FLAG_SAME_STEP_RESET; non-NULL
 *                 on another handle returns BSB_INVALID_ARGUMENT): the row of
 *                 each lane whose step_type is LAST receives the observation
 *                 the reference returned with that LAST timestep; the rows of
 *                 other lanes are left untouched.  Not through bsb_step_host
 *                 (BSB_UNSUPPORTED).
 */
typedef struct bsb_outputs {
  float* observation;
  float* reward;
  double* reward_f64;
  float* discount;
  int32_t* step_type;
  float* final_observation;
} bsb_outputs;

typedef struct bsb_env bsb_env; /* opaque handle */

int32_t bsb_abi_version(void);

/* Thread-local description of the last failure on the calling thread. */
const char* bsb_last_error(void);

/*
 * Replaces bsuite.load(name, kwargs) -> env constructor (bsuite/bsuite.py:93-98
 * and the constructors listed at bsb_family).  Creates `batch` lanes of one
 * environment; lane i has global id lane_offset + i (RNG keys depend on the
 * GLOBAL id only, so results are invariant to how lanes are sharded over GPUs).
 * Every lane starts with _reset_next_step = True (base.py:51-52) and performs
 * the constructor's RNG draws (memory_chain.py:49-50, umbrella_chain.py:55).
 * device >= 0: CUDA device ordinal; BSB_DEVICE_HOST: explicit host path.
 */
int32_t bsb_create(const bsb_config* config, int64_t batch, int32_t device,
                   uint64_t seed, uint64_t lane_offset, bsb_env** out);

/*
 * Packed handle: the settings of one experiment (bsuite_ids that share
 * everything that shapes the kernel and the observation) in ONE handle, so a
 * step of the whole experiment is one launch and one output tensor.  The
 * handle has batch B = n_settings * lanes_per_setting, and lane
 * k * lanes_per_setting + j of it is, bit for bit, lane j of
 *   bsb_create(&configs[k], lanes_per_setting, device, seeds[k], lane_offset)
 * -- its outputs, info, Logging columns, log rows, clamping of device actions,
 * and the actions bsb_rollout samples for it (keyed by lane_offset + j, the
 * lane within its setting).  Random streams therefore do not depend on the
 * packing, and a rank that owns lanes [a, b) of every setting creates its
 * pack with lanes_per_setting = b - a and lane_offset = a.
 * Settings may differ in their seed (seeds[k]; configs[k].seed is not a
 * field), the contents of `table` (bandit / discounting_chain rewards),
 * memory_length, chain_length, height_threshold, x_reward_threshold,
 * noise_scale and reward_scale; every other field must be equal, including
 * table sizes, mnist's images and labels and the log schedule
 * (BSB_UNSUPPORTED, naming the first field that differs).  n_settings in
 * [1, BSB_MAX_PACKED_SETTINGS] and lanes_per_setting >= 1, else
 * BSB_INVALID_ARGUMENT.  Not available (BSB_UNSUPPORTED): deep_sea (its
 * settings differ in size), BSB_RNG_MT19937, obs_dtype other than float32,
 * BSB_FLAG_SAME_STEP_RESET.  Every other entry point takes a packed handle as
 * a batch of B lanes; bsb_step_host runs it in one phase.
 */
int32_t bsb_create_packed(const bsb_config* configs, int32_t n_settings,
                          int64_t lanes_per_setting, int32_t device,
                          const uint64_t* seeds, uint64_t lane_offset,
                          bsb_env** out);

/* Settings and lanes per setting of a handle (1 and B for bsb_create's). */
int32_t bsb_packed_layout(const bsb_env* env, int32_t* n_settings,
                          int64_t* lanes_per_setting);

/*
 * Ragged pack: a packed handle whose settings differ in observation shape,
 * with the same contract as bsb_create_packed -- lane k * lanes_per_setting
 * + j is, bit for bit, lane j of
 *   bsb_create(&configs[k], lanes_per_setting, device, seeds[k], lane_offset)
 * (outputs, info, Logging columns, log rows, clamping of device actions and
 * the actions bsb_rollout samples).  Beyond what packs allow, settings may
 * differ in size together with the deep_sea mapping table, num_bits and
 * n_distractor.  Families: deep_sea, memory_chain, umbrella_chain (any other
 * returns BSB_UNSUPPORTED: use bsb_create_packed).  BSB_UNSUPPORTED, naming
 * the field: BSB_RNG_MT19937, obs_dtype other than float32,
 * BSB_FLAG_SAME_STEP_RESET, a reward wrapper, or a field the settings must
 * share.  n_settings in [1, BSB_MAX_PACKED_SETTINGS] and
 * lanes_per_setting >= 1, else BSB_INVALID_ARGUMENT.
 *
 * The observations of one step are ONE flat float32 buffer of step_elems
 * elements (bsb_ragged_layout; a rollout's is [T][step_elems]): setting k's
 * are a dense [lanes_per_setting, rows[k], cols[k]] block at element
 * offsets[k].  Blocks follow setting order, each starts on a 128-byte
 * boundary and step_elems is a multiple of 128 bytes; the gap elements
 * between blocks are never written.  bsb_outputs.observation and
 * bsb_step_host's device_obs / host_out->observation are that buffer;
 * final_observation is refused.  bsb_obs_numel / bsb_obs_shape return
 * BSB_UNSUPPORTED.  Every other entry point takes the handle as a batch of
 * B = n_settings * lanes_per_setting lanes, as for a pack; bsb_step_host runs
 * it in one phase.
 */
int32_t bsb_create_ragged(const bsb_config* configs, int32_t n_settings,
                          int64_t lanes_per_setting, int32_t device,
                          const uint64_t* seeds, uint64_t lane_offset,
                          bsb_env** out);

/* The observation buffer of a handle: offsets int64 [n_settings], rows and
 * cols int32 [n_settings] (n_settings of bsb_packed_layout) and the elements
 * of one step.  Every handle has one: an ordinary or uniformly packed handle
 * reports offsets k * lanes_per_setting * obs_numel and step_elems
 * B * obs_numel. */
int32_t bsb_ragged_layout(const bsb_env* env, int64_t* offsets, int32_t* rows,
                          int32_t* cols, int64_t* step_elems);

int32_t bsb_destroy(bsb_env* env);

/* observation_spec() / action_spec() (e.g. deep_sea.py:146-151). */
int32_t bsb_obs_numel(const bsb_env* env, int64_t* numel);
int32_t bsb_obs_shape(const bsb_env* env, int32_t* rows, int32_t* cols);
int32_t bsb_num_actions(const bsb_env* env, int32_t* num_actions);
int32_t bsb_batch(const bsb_env* env, int64_t* batch);

/* base.Environment.reset (base.py:54-57; cartpole.py:118-128): every lane
 * starts a new episode and emits FIRST. */
int32_t bsb_reset(bsb_env* env, const bsb_outputs* out, void* stream);

/* base.Environment.step (base.py:59-65) for all lanes; actions int32 [B]. */
int32_t bsb_step(bsb_env* env, const int32_t* actions, const bsb_outputs* out,
                 void* stream);

/*
 * Masked calls: reset() / step() for the lanes i with mask[i] != 0 only.
 * mask is uint8 [B] in the handle's memory space (device memory for a CUDA
 * handle, host memory for BSB_DEVICE_HOST).  An active lane makes exactly the
 * call bsb_reset / bsb_step would make for it (same transition, same random
 * draws, same outputs).  An inactive lane makes no call: its state, RNG
 * streams, info fields and Logging columns stay as they were, its action is
 * never read (so it never raises the invalid-action flag), and none of its
 * output entries -- observation row, reward, discount, step_type,
 * final_observation -- is written.  Lane i of a handle driven by masked calls
 * is, bit for bit, lane 0 of a one-lane handle with lane_offset + i driven by
 * the calls in which mask[i] was set.  Every masked call advances the call
 * count (bsb_steps_done) by one, even with an empty mask.  Works in
 * graph-safe mode and may be captured; a replay reads the mask buffer as it
 * is then.  Masked steps take explicit actions (int32 [B]) only.
 */
int32_t bsb_reset_masked(bsb_env* env, const uint8_t* mask,
                         const bsb_outputs* out, void* stream);
int32_t bsb_step_masked(bsb_env* env, const int32_t* actions,
                        const uint8_t* mask, const bsb_outputs* out,
                        void* stream);

/*
 * T consecutive step() calls fused in one launch, lane state held in
 * registers (replaces the inner loop of baselines/experiment.py:45-57).
 * actions: int32 [T,B], or NULL to sample uniform random actions on device
 * (the workload of baselines/random/agent.py:35-37) from the action stream
 * (action_seed, global lane, global step index) -- bsb_random_actions is its
 * host mirror.  actions_out (nullable) int32 [T,B] receives the actions used.
 * Outputs carry a leading T axis.
 */
int32_t bsb_rollout(bsb_env* env, int64_t num_steps, const int32_t* actions,
                    uint64_t action_seed, const bsb_outputs* out,
                    int32_t* actions_out, void* stream);

/*
 * Masked rollout: T masked steps fused in one launch, each lane stopping at
 * its own episode budget.  num_steps, actions (int32 [T,B] or NULL to sample
 * as bsb_rollout does at global step steps_done + t), action_seed, out
 * (leading T axis; final_observation on same-step handles) and actions_out
 * mean what they mean for bsb_rollout.  mask (uint8 [B], required) and
 * episodes_left (int64 [B], nullable) live in the handle's memory space.
 * Lane i is active at step t when mask[i] != 0 and episodes_left is NULL or
 * its budget left_i(t) > 0, where left_i(0) = episodes_left[i] and each LAST
 * timestep of an active step (a same-step handle's merged LAST included)
 * takes one from it; episodes_left[i] receives left_i(T).  A lane's active
 * steps are therefore a prefix of the T.  The call equals, bit for bit, T
 * calls of bsb_step_masked with mask_t[i] = active(i, t): every output entry
 * written, actions_out, lane state, RNG streams, info fields, Logging
 * columns, log rows, bsb_steps_done (+T) and the invalid-action flag.  The
 * (lane, t) entries of inactive steps -- in every output and in actions_out
 * -- are not written, and their actions are never read.  A host handle
 * refuses (BSB_INVALID_ARGUMENT, before anything moves) an out-of-range
 * action of any lane whose mask is set at ANY of the T steps, including
 * steps after its budget would have stopped it.  Works in graph-safe mode
 * and may be captured: a replay reads mask and episodes_left as they are
 * then and writes episodes_left back, so replays keep counting budgets down.
 */
int32_t bsb_rollout_masked(bsb_env* env, int64_t num_steps,
                           const int32_t* actions, uint64_t action_seed,
                           const uint8_t* mask, int64_t* episodes_left,
                           const bsb_outputs* out, int32_t* actions_out,
                           void* stream);

/*
 * Advance: a masked rollout of sampled actions that writes no per-step
 * output, for runs whose results live in the lanes' accumulators, log rows
 * and scores (playing every lane to its episode budget).  The call equals,
 * bit for bit, bsb_rollout_masked(env, num_steps, NULL, action_seed, mask,
 * episodes_left, out, NULL, stream) for any out, in everything but the
 * outputs: lane state, RNG streams (an observation's own draws, such as
 * umbrella_chain's distractors, are still made), info fields, Logging
 * columns, log rows, episodes_left and bsb_steps_done (+T).  Nothing per step
 * is written: no observation, final observation, scalar or action.  mask
 * (uint8 [B], required) and episodes_left (int64 [B], nullable) live in the
 * handle's memory space.  Refused (BSB_INVALID_ARGUMENT): a NULL env or mask,
 * num_steps <= 0.  Accepts every handle bsb_rollout_masked accepts, collects
 * an uncollected BSB_HOST_NO_WAIT step first, works in graph-safe mode and may
 * be captured: a replay reads mask and episodes_left as they are then and
 * writes episodes_left back.
 */
int32_t bsb_advance_masked(bsb_env* env, int64_t num_steps,
                           uint64_t action_seed, const uint8_t* mask,
                           int64_t* episodes_left, void* stream);

/*
 * Budgeted step: one masked step with episode budgets that first keeps the
 * outputs the agent acted on, so an agent loop needs one call per step.
 * For each lane i with mask[i] != 0: (1) lane i's current entries of `out`
 * -- observation row, reward, reward_f64, discount, step_type, and
 * final_observation when both output sets carry it -- are copied (as raw
 * bytes) to the same entries of `previous`, for each scalar both carry;
 * (2) if episodes_left[i] > 0 the lane makes exactly the call
 * bsb_rollout_masked(env, 1, actions, 0, mask, episodes_left, out, NULL,
 * stream) makes for it (a LAST takes one from its budget); (3) otherwise it
 * sits out and mask[i] is cleared.  Lanes whose mask is clear are not
 * touched.  So the call equals: copy out -> previous where mask; then that
 * bsb_rollout_masked; then mask[i] &= (episodes_left[i] > 0 before the
 * call) -- in outputs, previous, mask, budgets, lane state, RNG streams,
 * info fields, Logging columns, log rows, bsb_steps_done (+1) and the
 * invalid-action flag.  The mask is cleared one call AFTER the budget is
 * spent: on the call that returns a lane's last LAST, `previous` still holds
 * the timestep before it; on the next call both hold the LAST.  Actions of
 * lanes that sit out are never read.  actions (int32 [B]), mask (uint8 [B],
 * updated in place), episodes_left (int64 [B], counted down in place), out
 * and previous all live in the handle's memory space and are required.
 * Refused (BSB_INVALID_ARGUMENT): a NULL pointer (or observation buffer),
 * `previous` whose observation buffer is out's, final_observation set in one
 * output set and not the other, final_observation on a next-step handle.
 * Accepts every handle bsb_step_masked accepts, collects an uncollected
 * BSB_HOST_NO_WAIT step first, works in graph-safe mode and may be captured:
 * a replay reads and writes mask and episodes_left as they are then.
 */
int32_t bsb_step_budgeted(bsb_env* env, const int32_t* actions, uint8_t* mask,
                          int64_t* episodes_left, const bsb_outputs* out,
                          const bsb_outputs* previous, void* stream);

/*
 * Policy step: bsb_step_budgeted where the engine chooses each lane's action
 * from the agent's network output, so a learning agent's epsilon-greedy or
 * softmax selection needs no kernels of its own.  The call equals
 * bsb_step_budgeted(env, A, mask, episodes_left, out, previous, stream), bit
 * for bit, where A holds the actions the policy picks; actions_out (int32
 * [B], nullable) receives A[i] for every lane that stepped (mask set, budget
 * left).  Other lanes' entries are not written and their value rows are
 * never read.
 *
 * The policy stream: lane i's draw is the Philox4x64-10 block at counter
 * (s, 0, 0, 3), s being the call's global step index (the step0 bsb_rollout
 * samples at), with key (seed, global lane) -- keyed as bsb_rollout keys its
 * sampled actions, so in a pack it is the lane within its setting.  Its words
 * w0, w1 are all a lane uses.  It is stateless: nothing enters the state
 * snapshot.
 *   EPSILON_GREEDY: u = (w0 >> 11) * 2^-53; u < epsilon explores and picks
 *     (lo32(w1) * A) >> 32.  Otherwise, with k entries equal (float ==) to
 *     the row's maximum, the pick is the ((lo32(w1) * k) >> 32)-th of them in
 *     ascending order.  +-inf are ordinary values.
 *   SOFTMAX: w_a = exp((double)l_a - max) (-inf weighs 0), computed by an
 *     exp the host path and the kernels share; target = ((w1 >> 11) *
 *     2^-53) * sum(w).  The pick is the first a whose running double sum
 *     exceeds the target, or the last a of positive weight if none does.
 * A row containing NaN, or for SOFTMAX a row containing +inf or without a
 * finite entry, raises the invalid-action flag (bsb_invalid_actions; host
 * handles too) and that lane picks (lo32(w1) * A) >> 32.
 * Refused (BSB_INVALID_ARGUMENT, before anything moves): whatever
 * bsb_step_budgeted refuses, a NULL policy or values, an unknown kind, a
 * non-zero `reserved`, epsilon outside [0, 1] or NaN, a non-zero epsilon for
 * SOFTMAX.  values (float32 [B, A], contiguous) and actions_out live in the
 * handle's memory space.  Accepts every handle bsb_step_budgeted accepts and
 * may be captured: a replay reads values, mask and budgets as they are then,
 * while kind, epsilon and seed replay as captured.
 */
typedef enum bsb_policy_kind { BSB_POLICY_EPSILON_GREEDY = 0, BSB_POLICY_SOFTMAX = 1 } bsb_policy_kind;
typedef struct bsb_policy {
  int32_t kind;          /* bsb_policy_kind */
  int32_t reserved;      /* 0 */
  const float* values;   /* float32 [B, num_actions], contiguous, in the handle's memory space:
                            action values (EPSILON_GREEDY) or logits (SOFTMAX) */
  double epsilon;        /* EPSILON_GREEDY: in [0, 1]; SOFTMAX: must be 0 */
  uint64_t seed;         /* key of the policy stream */
} bsb_policy;

int32_t bsb_step_budgeted_policy(bsb_env* env, const bsb_policy* policy, uint8_t* mask,
                                 int64_t* episodes_left, const bsb_outputs* out,
                                 const bsb_outputs* previous, int32_t* actions_out, void* stream);

/*
 * Per-lane replay rings (baselines/replay.py, one ring per lane, as each
 * bsuite_id run of the reference owns its own replay).  The layout is the
 * engine's [T, B, ...] rollout layout with T = capacity: obs_tm1 and
 * next.observation are [capacity][step_elems] in the handle's obs_dtype (raw
 * bytes, cast as for bsb_outputs; a ragged pack's settings at the offsets
 * bsb_ragged_layout reports), action / next.reward / next.reward_f64 /
 * next.discount / next.step_type are [capacity, B].  Offsets are 64-bit.
 * next.final_observation is always NULL.  In a batch written by
 * bsb_replay_sample, capacity is the sample size and num_added is NULL.
 */
typedef struct bsb_replay {
  int64_t capacity;        /* slots per lane, in [1, 2^31 - 1] */
  int64_t* num_added;      /* int64 [B]: transitions added per lane; NULL in a sample's output */
  float* obs_tm1;          /* [capacity][step_elems] in the handle's obs_dtype */
  int32_t* action;         /* int32 [capacity, B] */
  bsb_outputs next;        /* o_t / r_t / d_t / step_type with a leading capacity axis (scalars nullable) */
} bsb_replay;

/*
 * Recorded step: bsb_step_budgeted (actions != NULL) or
 * bsb_step_budgeted_policy (policy != NULL; exactly one of the two) that also
 * appends each transition to its lane's ring.  The call equals that call bit
 * for bit in everything it defines.  In addition every lane that stepped
 * (mask set and episodes_left > 0 before the call) and whose new step_type
 * is not FIRST writes slot c = num_added[i] % capacity of its ring, then
 * num_added[i] += 1 (replay.py:51-54):
 *   obs_tm1[c]            the observation row copied to `previous`
 *   action[c, i]          the action used (the caller's action after
 *                         clamping, or the policy's pick)
 *   next.reward[c, i]     the new reward, in whichever of float32 / float64
 *                         the ring carries (cast from out's if out carries the
 *                         other one); next.discount, next.step_type likewise
 *   next.observation[c]   the new observation row; on a same-step handle whose
 *                         new step_type is LAST, the final observation row.
 * Lanes that only restarted (new FIRST) or sat out write nothing.  The rows
 * are copied, never re-rendered.  out->step_type is required (it decides
 * FIRST), and a same-step handle must pass out->final_observation.
 * Refused (BSB_INVALID_ARGUMENT, before anything moves): whatever the
 * underlying budgeted or policy step refuses, both or neither of actions and
 * policy, a NULL replay / num_added / obs_tm1 / action / next.observation or
 * out->step_type, a ring reward with no reward in `out`, capacity outside
 * [1, 2^31 - 1], a ring observation buffer that is out's or previous's,
 * next.final_observation non-NULL, a same-step handle without
 * out->final_observation.  Every handle bsb_step_budgeted accepts; graph-safe
 * mode and capture included: a replay reads and writes num_added as it is
 * then.
 */
int32_t bsb_step_budgeted_record(bsb_env* env, const int32_t* actions, const bsb_policy* policy,
                                 uint8_t* mask, int64_t* episodes_left,
                                 const bsb_outputs* out, const bsb_outputs* previous,
                                 int32_t* actions_out, const bsb_replay* replay, void* stream);

/*
 * Uniform minibatches from every lane's ring, in one launch.  For every lane
 * i with n = min(capacity, num_added[i]) >= max(min_size, 1), batch slot j
 * in [0, size) receives ring slot s_j = (lo32(w) * n) >> 32 of lane i --
 * obs_tm1, action and each of next's fields that both `replay` and `batch`
 * carry -- where w is word (j & 3) of the Philox4x64-10 block at counter
 * (c, draw, j >> 2, 4) with key (seed, global lane).  c is the handle's
 * current call index (bsb_steps_done; in graph-safe mode read on the device,
 * so a captured sample draws fresh slots at every replay), `draw` tells apart
 * several samples between two calls, and the global lane is keyed as the
 * policy stream keys it (in a pack: the lane within its setting), so shards,
 * packs and standalone handles draw the same slots.  ready[i] (uint8 [B],
 * nullable) is set to 1 for these lanes and 0 for the others, whose batch
 * entries are not written (replay.py: `if size < min_replay_size: return`).
 * The gather moves raw bytes.  Refused (BSB_INVALID_ARGUMENT): size <= 0,
 * min_size < 0, a NULL replay / num_added / obs_tm1 / action /
 * next.observation, or batch / obs_tm1 / action / next.observation, a batch
 * whose capacity != size or whose num_added is non-NULL, a ring capacity out
 * of range, a batch scalar the ring does not carry.
 */
int32_t bsb_replay_sample(bsb_env* env, const bsb_replay* replay, int64_t size, int64_t min_size,
                          uint64_t seed, uint64_t draw, const bsb_replay* batch, uint8_t* ready,
                          void* stream);

/*
 * Per-lane sequence buffers (baselines/utils/sequence.py's Buffer, one
 * window of at most T = max_length transitions per lane, as the reference's
 * actor_critic and actor_critic_rnn keep one per bsuite_id run).  The layout
 * is the engine's rollout layout: observations is [T + 1][step_elems] in the
 * handle's obs_dtype (raw bytes, a ragged pack's settings at the offsets
 * bsb_ragged_layout reports), action / next.reward / next.reward_f64 /
 * next.discount / next.step_type are [T, B].  Offsets are 64-bit.  Lane i's
 * current sequence is observations[0 .. length[i]] and entries
 * [0, length[i]) of the others; later entries are stale.
 */
typedef struct bsb_sequence {
  int64_t max_length;      /* T, in [1, 2^31 - 1] */
  int64_t* length;         /* int64 [B]: transitions in the lane's current sequence */
  uint8_t* ready;          /* uint8 [B]: written for every lane by every call */
  float* observations;     /* [T + 1][step_elems] in the handle's obs_dtype */
  int32_t* action;         /* int32 [T, B] */
  bsb_outputs next;        /* reward or reward_f64, discount, step_type [T, B];
                              observation and final_observation NULL */
} bsb_sequence;

/*
 * Sequence step: bsb_step_budgeted (actions != NULL) or
 * bsb_step_budgeted_policy (policy != NULL; exactly one of the two) that also
 * appends each transition to its lane's sequence.  The call equals that call
 * bit for bit in everything it defines.  In addition every lane i that
 * stepped (mask set and episodes_left > 0 before the call) and whose new
 * step_type is not FIRST appends one transition (sequence.py's append):
 *   t = length[i]; if t == T, or t > 0 and next.step_type[t - 1, i] is LAST,
 *   the previous sequence was drained: t = 0 (a length outside [0, T) also
 *   starts over)
 *   observations[0]       (t == 0 only) the observation row copied to
 *                         `previous`: o_tm1, what the agent acted on
 *   observations[t + 1]   the new observation row; on a same-step handle whose
 *                         new step_type is LAST, the final observation row
 *   action[t, i]          the action used (the caller's action after
 *                         clamping, or the policy's pick)
 *   next.*[t, i]          the new reward (cast as bsb_step_budgeted_record
 *                         casts it), discount and step_type
 *   length[i] = t + 1, ready[i] = (t + 1 == T or the new step_type is LAST).
 * Every other lane gets ready[i] = 0 and nothing else is written, so `ready`
 * marks exactly the sequences this call closed (sequence.py: `if full() or
 * last(): drain()`); the drain happens lazily at the lane's next append, so
 * the closed sequence can be read until the next call.  The rows are copied,
 * never re-rendered.  State lives in `length` and next.step_type only.
 * Refused (BSB_INVALID_ARGUMENT, before anything moves): whatever the
 * underlying budgeted or policy step refuses, both or neither of actions and
 * policy, actions_out with actions, a NULL sequence / length / ready /
 * observations / action / next.step_type / next.discount, both rewards
 * NULL, a sequence reward with no reward in `out`, max_length outside
 * [1, 2^31 - 1], next.observation or next.final_observation non-NULL, an
 * observation buffer that is out's or previous's, out->step_type NULL, a
 * same-step handle without out->final_observation.  Every handle
 * bsb_step_budgeted accepts; graph-safe mode and capture included.
 */
int32_t bsb_step_budgeted_sequence(bsb_env* env, const int32_t* actions, const bsb_policy* policy,
                                   uint8_t* mask, int64_t* episodes_left,
                                   const bsb_outputs* out, const bsb_outputs* previous,
                                   int32_t* actions_out, const bsb_sequence* sequence, void* stream);

/*
 * Ensemble policy (the reference's boot_dqn, baselines/jax/boot_dqn/agent.py:
 * one ensemble member acts per episode, epsilon-greedily over its Q-values).
 * values holds every head's action values; heads holds each lane's active
 * head, which the caller zero-fills before a run (the reference starts on
 * member 0) and the step redraws when an episode ends.
 */
typedef struct bsb_ensemble_policy {
  int32_t num_heads;     /* K, in [1, 65536] */
  int32_t reserved;      /* 0 */
  const float* values;   /* float32 [K, B, num_actions], contiguous: every head's action values */
  int32_t* heads;        /* int32 [B]: each lane's active head; read, and redrawn at a LAST */
  double epsilon;        /* in [0, 1] */
  uint64_t seed;         /* keys the policy stream and the head stream */
} bsb_ensemble_policy;

/*
 * Ensemble step.  Let h_i = heads[i] before the call and V the [B, A] rows
 * values[h_i, i, :].  With replay == NULL the call equals
 * bsb_step_budgeted_policy with {EPSILON_GREEDY, V, epsilon, seed} bit for
 * bit (outputs, previous, actions_out, mask, budgets, lane state, streams,
 * info, Logging columns, log rows, step count); with a replay it equals
 * bsb_step_budgeted_record with that policy, rings included.  In addition
 * every lane that stepped (mask set and episodes_left > 0 before the call)
 * and whose step ended an episode (the LAST that counts its budget down; no
 * output is read for it) sets heads[i] = (lo32(w0) * K) >> 32 (update(),
 * agent.py:166-169), w0 being word 0 of the Philox4x64-10 block at counter
 * (s, 0, 0, 5) with key (seed, global lane): s and the global lane are those
 * of the policy stream.  Lanes that sit out read no row and keep their head.
 * A head outside [0, K) raises the invalid-action flag and is clamped for
 * the row read, as actions are; it is not written back.
 * Refused (BSB_INVALID_ARGUMENT, before anything moves): whatever
 * bsb_step_budgeted_policy or bsb_step_budgeted_record refuses, a NULL
 * policy / values / heads, num_heads outside [1, 65536], a non-zero
 * `reserved`, epsilon outside [0, 1] or NaN.  values and heads live in the
 * handle's memory space.  May be captured: a replay reads values, heads,
 * mask and budgets as they are then.
 */
int32_t bsb_step_budgeted_ensemble(bsb_env* env, const bsb_ensemble_policy* policy, uint8_t* mask,
                                   int64_t* episodes_left, const bsb_outputs* out,
                                   const bsb_outputs* previous, int32_t* actions_out,
                                   const bsb_replay* replay, void* stream);

/*
 * Bootstrap masks and reward noise of boot_dqn's transitions
 * (agent.py:171-185: m_t ~ Bernoulli(mask_prob)^K, z_t ~ N(0, 1)^K per
 * transition), drawn when a transition is sampled rather than stored.  Each is
 * a pure function of (seed, global lane, j), j being the 0-based count of
 * transitions the lane had added before this one, so a transition keeps its
 * draws however often it is sampled.  mask and noise are [size, B, K] in the
 * handle's memory space; either may be NULL, not both.
 */
typedef struct bsb_bootstrap {
  int32_t num_heads;     /* K, in [1, 65536] */
  int32_t reserved;      /* 0 */
  double mask_prob;      /* in [0, 1] */
  uint64_t seed;         /* key of the bootstrap stream */
  uint8_t* mask;         /* uint8 [size, B, K], nullable */
  float* noise;          /* float32 [size, B, K], nullable */
} bsb_bootstrap;

/*
 * bsb_replay_sample with bootstrap draws: the call equals bsb_replay_sample
 * bit for bit.  In addition, for every entry (j', i) it writes for a ready
 * lane, with slot the ring slot it drew, N = num_added[i] and
 * j = N - 1 - ((N - 1 - slot) mod capacity) the transition's index, and for
 * every head k, on the Philox4x64-10 blocks with key (bootstrap->seed, global
 * lane) (the global lane keyed as the sample keys it):
 *   mask[j', i, k] = ((w >> 11) * 2^-53 < mask_prob), w = word k & 3 of the
 *     block at counter (j, k >> 2, 0, 6);
 *   noise[j', i, k] = numpy's legacy polar method on the blocks at counter
 *     (j, k, 1 + a, 6), a = 0, 1, ...: x = 2 (w0 >> 11) 2^-53 - 1, y likewise
 *     from w1, accepted when 0 < r2 = x^2 + y^2 < 1, noise = (float)(y *
 *     sqrt(-2 log(r2) / r2)) with a log the host path and the kernels share;
 *     0 after 64 rejected attempts (probability below 1e-42).
 * Entries of other lanes are not written.  Refused (BSB_INVALID_ARGUMENT):
 * whatever bsb_replay_sample refuses, a NULL bootstrap, num_heads outside
 * [1, 65536], a non-zero `reserved`, mask_prob outside [0, 1] or NaN, mask
 * and noise both NULL.  May be captured, as bsb_replay_sample.
 */
int32_t bsb_replay_sample_bootstrap(bsb_env* env, const bsb_replay* replay, int64_t size, int64_t min_size,
                                    uint64_t seed, uint64_t draw, const bsb_replay* batch, uint8_t* ready,
                                    const bsb_bootstrap* bootstrap, void* stream);

/* Host mirror of the on-device action sampler: out int32 [T,B] (host). */
int32_t bsb_random_actions(uint64_t action_seed, uint64_t lane_offset,
                           int64_t batch, int64_t first_step, int64_t num_steps,
                           int32_t num_actions, int32_t* out);

/* Number of step()/reset() calls made so far (global step index). */
int32_t bsb_steps_done(const bsb_env* env, int64_t* steps);

/*
 * bsuite_info() (e.g. deep_sea.py:153-155): per-lane accumulators.
 * bsb_info_count / bsb_info_name enumerate the keys of the reference dict;
 * bsb_read_info copies field `index` as float64 [B] into dst (same memory
 * space as the environment).
 */
int32_t bsb_info_count(const bsb_env* env, int32_t* count);
const char* bsb_info_name(const bsb_env* env, int32_t index);
int32_t bsb_read_info(bsb_env* env, int32_t index, double* dst, void* stream);

/*
 * Logging-wrapper accumulators (utils/wrappers.py:85-110), kept per lane when
 * BSB_FLAG_TRACK_EPISODES is set: field 0 steps, 1 episode, 2 total_return,
 * 3 episode_len, 4 episode_return; float64 [B] each.  episode_len and
 * episode_return are zeroed when the NEXT episode starts, so from a LAST
 * timestep (when the reference writes its row, :99-101) until the lane steps
 * again they hold the finished episode's values.
 */
int32_t bsb_read_episode_stats(bsb_env* env, int32_t field, double* dst,
                               void* stream);

/*
 * CUDA graphs.  bsb_step / bsb_reset / bsb_rollout / the masked calls (bsb_reset_masked / bsb_step_masked /
 * bsb_rollout_masked / bsb_advance_masked / bsb_step_budgeted / bsb_step_budgeted_policy / bsb_step_budgeted_record
 * / bsb_step_budgeted_sequence / bsb_step_budgeted_ensemble) / bsb_replay_sample / bsb_replay_sample_bootstrap /
 * bsb_read_* / bsb_sum_* may
 * be called on a stream that is being captured.  A graph freezes launch arguments, so the first captured launch moves the handle's step
 * counter (it indexes the on-device action stream and the Logging columns) and its chunk scheduler into device
 * memory, for good: replays and eager calls can then be mixed in any order, and bsb_steps_done / bsb_get_state
 * synchronise the device to read the counter back.  Consecutive captured steps keep their programmatic dependent
 * launch (it becomes a programmatic graph edge).
 * bsb_step_host (internal stream, host-side wait) cannot be captured.
 */

/*
 * Device-side reduction of the same five columns over the lanes of this
 * environment: dst[5] (same memory space as the environment) receives the SUMS
 * of steps, episode, total_return, episode_len, episode_return -- one small
 * kernel, so a log point costs a 40-byte read (or a 40-byte all-gather across
 * ranks) instead of five per-lane arrays.
 */
int32_t bsb_sum_episode_stats(bsb_env* env, double* dst5, void* stream);

/* The same reduction for `count` environments of one device in ONE kernel launch:
 * dst receives [count][5].  A log point of a whole sweep (bsuite/sweep.py:134-150:
 * 23 experiments) is then one launch and one all-gather.  Each handle may appear
 * once: a repeated handle returns BSB_INVALID_ARGUMENT on the host and the device
 * path alike (the launch keeps its partial sums in per-handle scratch). */
int32_t bsb_sum_episode_stats_many(bsb_env* const* envs, int32_t count,
                                   double* dst, void* stream);

/* Per-setting rows of the same reduction: dst receives [rows][5] (steps, episode,
 * total_return, episode_len, episode_return), rows in handle order and, within a
 * packed or ragged handle (bsb_create_packed / bsb_create_ragged), in setting
 * order; an ordinary handle gives one row, equal to bsb_sum_episode_stats.
 * Row k of a pack of L lanes per setting sums lanes [k*L, (k+1)*L) in the order a
 * standalone L-lane handle sums its own, so it equals, bit for bit,
 * bsb_sum_episode_stats of a standalone handle of that setting (its seed, L lanes,
 * the pack's lane_offset) after the same calls -- on the device and on the host
 * path alike.  Up to 64 handles (and every setting in them) take ONE launch; a
 * longer list takes one launch per handle.  Every setting has its own partials and
 * ticket, allocated with the handle.  Refusals as for bsb_sum_episode_stats_many.
 * May be captured in a CUDA graph; graph-safe handles read their step counter on
 * the device. */
int32_t bsb_sum_setting_stats(bsb_env* const* envs, int32_t count,
                              double* dst, void* stream);

/*
 * Per-lane log rows (see bsb_config.log_schedule): row k of lane i holds the
 * reference wrapper's columns steps, episode, total_return, episode_len,
 * episode_return followed by the bsuite_info() fields (bsb_info_name order) at
 * the LAST timestep that completed episode log_schedule[k] of that lane.
 * bsb_log_layout reports [n_points, n_columns]; bsb_read_log_rows copies
 * rows float64 [n_points][n_columns][B] and counts int32 [B] (rows recorded so
 * far per lane) into caller buffers in the environment's memory space.
 */
int32_t bsb_log_layout(const bsb_env* env, int32_t* n_points, int32_t* n_columns);
int32_t bsb_read_log_rows(bsb_env* env, double* rows, int32_t* counts, void* stream);

/*
 * bsuite scores from the log rows (experiments/summary_analysis.py:111-171,
 * bsuite_score and ave_score_by_tag, on the results directory of each lane).
 * Lane j of every source is one run of the sweep, as lane j's directory of
 * CSV files (recording.write_lane_csvs) is for the reference: scores[e][j]
 * is the score experiment e gets from those files, finished[e][j] whether
 * each of its settings present reached NUM_EPISODES, and tag_scores[t][j]
 * the mean over the experiments tagged t (NaN scores skipped).  An
 * experiment with no row at lane j scores NaN and is not finished.
 * Experiments are numbered in sorted name order and tags in sorted tag order.
 */
typedef enum bsb_experiment {
  BSB_EXP_BANDIT = 0, BSB_EXP_BANDIT_NOISE, BSB_EXP_BANDIT_SCALE,
  BSB_EXP_CARTPOLE, BSB_EXP_CARTPOLE_NOISE, BSB_EXP_CARTPOLE_SCALE,
  BSB_EXP_CARTPOLE_SWINGUP, BSB_EXP_CATCH, BSB_EXP_CATCH_NOISE,
  BSB_EXP_CATCH_SCALE, BSB_EXP_DEEP_SEA, BSB_EXP_DEEP_SEA_STOCHASTIC,
  BSB_EXP_DISCOUNTING_CHAIN, BSB_EXP_MEMORY_LEN, BSB_EXP_MEMORY_SIZE,
  BSB_EXP_MNIST, BSB_EXP_MNIST_NOISE, BSB_EXP_MNIST_SCALE,
  BSB_EXP_MOUNTAIN_CAR, BSB_EXP_MOUNTAIN_CAR_NOISE,
  BSB_EXP_MOUNTAIN_CAR_SCALE, BSB_EXP_UMBRELLA_DISTRACT,
  BSB_EXP_UMBRELLA_LENGTH, BSB_NUM_EXPERIMENTS
} bsb_experiment;

typedef enum bsb_tag {
  BSB_TAG_BASIC = 0, BSB_TAG_CREDIT_ASSIGNMENT, BSB_TAG_EXPLORATION,
  BSB_TAG_GENERALIZATION, BSB_TAG_MEMORY, BSB_TAG_NOISE, BSB_TAG_SCALE,
  BSB_NUM_TAGS
} bsb_tag;

/* The row columns a score reads: bsb_score_source.columns[quantity]. */
typedef enum bsb_score_quantity {
  BSB_Q_EPISODE = 0, BSB_Q_TOTAL_RETURN, BSB_Q_TOTAL_REGRET,
  BSB_Q_RAW_RETURN, BSB_Q_BEST_EPISODE, BSB_Q_TOTAL_PERFECT,
  BSB_Q_TOTAL_BAD_EPISODES, BSB_SCORE_NUM_QUANTITIES
} bsb_score_quantity;

#define BSB_SCORE_MAX_SOURCES 512

/*
 * One setting (bsuite_id) of one experiment: its rows, read in place.
 *   env != NULL: the rows a handle created with a log schedule keeps
 *       (bsb_read_log_rows' layout; any host step still in flight is
 *       drained first).  rows, counts, n_points, n_columns, lane_stride and
 *       device are then ignored.
 *   env == NULL: caller-owned rows float64 [n_points][n_columns][lane_stride]
 *       and counts int32 [lane_stride] in the memory space `device`.
 * Lanes [first_lane, first_lane + lanes) of the store are lanes 0 .. lanes-1
 * of the result (a packed handle's setting k starts at k * lanes_per_setting).
 * `setting` is the index of the bsuite_id within its experiment, `group_key`
 * the sweep value the experiment groups by (noise_scale, reward_scale, size,
 * memory_length, num_bits, chain_length, n_distractor, height_threshold; 0
 * when it groups by none), and columns[q] the column holding quantity q, or
 * -1.  Rows must be recorded at strictly ascending episodes no larger than
 * the experiment's NUM_EPISODES, as every handle's log schedule is.
 */
typedef struct bsb_score_source {
  bsb_env* env;
  const double* rows;
  const int32_t* counts;
  int32_t n_points, n_columns;
  int64_t lane_stride;
  int32_t device;
  int32_t experiment;   /* bsb_experiment */
  int32_t setting;
  int32_t reserved0;
  int64_t first_lane, lanes;
  double group_key;
  int32_t columns[BSB_SCORE_NUM_QUANTITIES];
  int32_t reserved1;
} bsb_score_source;

/*
 * Scores `count` sources (any order, at most BSB_SCORE_MAX_SOURCES, each
 * setting once, all with `lanes` lanes and on one device) into scores
 * float64 [BSB_NUM_EXPERIMENTS][lanes], finished uint8 [BSB_NUM_EXPERIMENTS]
 * [lanes] (0 / 1) and tag_scores float64 [BSB_NUM_TAGS][lanes], all in the
 * sources' memory space.  A device call enqueues two kernels on `stream`
 * (one lane per thread and experiment, then the tag means) and neither
 * allocates nor synchronises; a host call is synchronous.  The rows are only
 * read.  BSB_INVALID_ARGUMENT: a handle without a log schedule, differing
 * lane counts or devices, an unknown experiment, a column the experiment's
 * score needs that is missing or out of range, a setting given twice.
 */
int32_t bsb_score(const bsb_score_source* sources, int32_t count, int64_t lanes,
                  double* scores, uint8_t* finished, double* tag_scores,
                  void* stream);

/* Flat snapshot of all lane state (checkpoint/resume; absent in the reference). */
int32_t bsb_state_bytes(const bsb_env* env, int64_t* nbytes);
int32_t bsb_get_state(bsb_env* env, void* dst_host, int64_t nbytes, void* stream);
int32_t bsb_set_state(bsb_env* env, const void* src_host, int64_t nbytes,
                      void* stream);

/*
 * Host-buffer convenience for FFI callers without a device allocator: takes
 * `actions` (host, int32 [B]), steps, and delivers the requested outputs into
 * HOST buffers (`host_out`; NULL members are skipped, so an agent that consumes
 * observations on the device passes observation = NULL and supplies
 * `device_obs`, a device pointer that receives them).  Synchronous for the
 * host outputs: on return they have landed (for `device_obs` see
 * BSB_HOST_FENCE_CALLER).  This
 * is the call pattern of the reference's agent loop, one env.step(action) per
 * decision (baselines/experiment.py:45-57).
 *
 * When `actions` and the requested scalar outputs are PINNED host memory the
 * kernel accesses them in place over PCIe (zero-copy: no separate H2D / D2H
 * copies) and signals completion through a pinned mailbox word the host spins
 * on (no stream synchronise); pageable buffers
 * take the staged-copy path.  Host actions are range-checked: an action outside
 * [0, num_actions) yields BSB_INVALID_ARGUMENT (the reference raises IndexError,
 * e.g. bandit.py:61).
 *
 * flags
 *   BSB_HOST_ORDER_AFTER_STREAM  work enqueued EARLIER on this handle through
 *       bsb_reset / bsb_step / bsb_rollout on `caller_stream` is waited for (on
 *       the device) before the step runs.  Without the flag the caller must
 *       have synchronised that stream: the step runs on a stream the handle owns.
 *   BSB_HOST_FENCE_CALLER  deep_sea from size 16 up (its observation is a function
 *       of the lane state and dwarfs the scalar traffic) runs host steps in two
 *       phases: the transitions of all lanes first (scalars staged on the device
 *       and shipped to the host by a few copier blocks), then the observation
 *       stream.  The call returns as soon as the scalars have landed -- the agent
 *       decides its next action while the observations are still being written.  With this flag `caller_stream`
 *       is fenced (on the device) behind the step, so work enqueued there
 *       afterwards sees complete observations; without it, order a consumer by
 *       the next call on this handle (every entry point waits for the step).
 *       Same-step handles (BSB_FLAG_SAME_STEP_RESET) always run host steps in
 *       one phase.
 *   BSB_HOST_PRELAUNCH  accepted, no effect: the call runs the same waited step
 *       as without it.  The mode it named (the next step's kernel queued ahead,
 *       polling a doorbell in pinned memory) was retired because it lost to the
 *       waited step on the H100.
 *   BSB_HOST_NO_WAIT  (pinned buffers; otherwise the call is simply synchronous)
 *       the call returns once the step is enqueued; the host outputs are valid
 *       after bsb_host_wait(env).  One step per handle may be outstanding (any
 *       entry point of the handle collects it first).  The use: split the lanes
 *       over TWO handles (bsb_create's lane_offset keeps the lanes' random streams
 *       those of one big batch) and alternate -- while one half's scalars cross
 *       PCIe and its agent decides, the other half's kernel has the GPU, so each
 *       half remains the reference's strict loop (act on what the previous step
 *       returned) and the GPU is not left idle in between (two to four handles).
 *       Pass BSB_HOST_FENCE_CALLER with it: without the fence's event record between
 *       a handle's consecutive launches, the next launch becomes a programmatic
 *       dependent of the previous one, parks its CTAs behind the other handles'
 *       work and the loop slows down.  Not with BSB_HOST_PRELAUNCH.
 */
#define BSB_HOST_ORDER_AFTER_STREAM 1u
#define BSB_HOST_PRELAUNCH 2u
#define BSB_HOST_FENCE_CALLER 4u
#define BSB_HOST_NO_WAIT 8u
int32_t bsb_step_host(bsb_env* env, const int32_t* actions,
                      const bsb_outputs* host_out, float* device_obs,
                      void* caller_stream, uint32_t flags);

/*
 * Masked host-driven step: bsb_step_host for a chosen subset of lanes, each
 * stopping at its own episode budget, so that a host-side agent can play every
 * lane to exactly its budget on the host step's fast path.  actions, host_out,
 * device_obs, caller_stream and flags mean what they mean for bsb_step_host
 * (BSB_HOST_NO_WAIT with bsb_host_wait / bsb_host_flush included; one step in
 * flight per handle; masked and unmasked host steps may be interleaved).
 *
 * mask (uint8 [B], required) lives in HOST memory, like actions: pinned memory
 * is read in place, pageable memory is staged.  episodes_left (int64 [B],
 * nullable) lives in the handle's memory space, as for bsb_rollout_masked
 * (device memory for a CUDA handle: budgets never cross PCIe).  Lane i is
 * active when mask[i] != 0 and episodes_left is NULL or episodes_left[i] > 0.
 * The call equals, bit for bit, bsb_rollout_masked(env, 1, actions, 0, mask',
 * episodes_left, out, NULL) with mask' a device copy of mask taken before the
 * call (without episodes_left: bsb_step_masked): every output entry written,
 * lane state, RNG streams, info fields, Logging columns, log rows,
 * episodes_left, bsb_steps_done (+1) and the invalid-action flag.  Inactive
 * lanes' entries of host_out's scalars and of device_obs are not written and
 * their actions are never read.  host_out->observation, when set, receives the
 * whole device observation buffer after the step.
 *
 * Mask write-back: with episodes_left, the call clears mask[i] in place for
 * every lane whose budget is <= 0 after the step, so that afterwards
 * mask[i] == old_mask[i] && episodes_left[i] > 0: the host always holds the set
 * of lanes still running.  Only lanes that just ran out (or whose budget was
 * already spent) write their byte, before the completion word (with
 * BSB_HOST_NO_WAIT: read the mask after bsb_host_wait).  Without
 * episodes_left the mask is only read.
 *
 * A masked host step always runs in one phase (its kernel has no bulk stores,
 * so completion means the observations are written), on deep_sea from size 16
 * up and catch too.  An out-of-range action of an active lane is refused before
 * anything moves on a host handle (BSB_INVALID_ARGUMENT); on a CUDA handle it is
 * clamped and reported after the step (BSB_INVALID_ARGUMENT, or by
 * bsb_host_wait), as bsb_step_host's zero-copy path does.  Refused:
 * final_observation (BSB_UNSUPPORTED) and a NULL mask.
 */
int32_t bsb_step_host_masked(bsb_env* env, const int32_t* actions,
                             uint8_t* mask, int64_t* episodes_left,
                             const bsb_outputs* host_out, float* device_obs,
                             void* caller_stream, uint32_t flags);

/* Collects a BSB_HOST_NO_WAIT step nobody waited for (no-op otherwise).  Unlike
 * bsb_host_wait it does not report an out-of-range action of that step. */
int32_t bsb_host_flush(bsb_env* env);

/* Completes a step issued with BSB_HOST_NO_WAIT: returns when its host outputs
 * have landed (no-op when nothing is outstanding).  Reports an out-of-range
 * action of that step as BSB_INVALID_ARGUMENT, like the synchronous call. */
int32_t bsb_host_wait(bsb_env* env);

/* Diagnostics (BSB_HOST_TIMING=1): %globaltimer stamps, in ns, the latest two-phase
 * host step left in the mailbox: [0] kernel past its dependency wait, [1] phase 1
 * complete, [2] scalars fenced, [3] latest block exit of the previous launch. */
int32_t bsb_host_timing(bsb_env* env, uint64_t* stamps8);

/*
 * Out-of-range actions.  Host-resident actions (host environments,
 * bsb_step_host) are validated before anything moves.  Device-resident action
 * tensors cannot be inspected without a synchronise: the kernels clamp such an
 * action into [0, num_actions) before it indexes a table or is packed into lane
 * state, and raise a flag.  *seen receives the flag (1 = some action since the
 * last call was out of range) and clears it; synchronise the stream first.
 */
int32_t bsb_invalid_actions(bsb_env* env, int32_t* seen);

/*
 * Multi-GPU log points without torch.distributed (SURVEY.md 8e: "one collective:
 * ncclAllGather of a per-rank stats block at log points only").  One process per
 * GPU; rank 0 calls bsb_comm_unique_id and shares the 128 bytes out of band (a
 * file, a socket, MPI, torch's store), every rank calls bsb_comm_create.  NCCL is
 * loaded at run time (BSB_NCCL_LIBRARY, else libnccl.so.2): single-GPU callers
 * never need it.
 *
 * bsb_log_point: the Logging sums of `count` environments of this rank are
 * reduced by ONE kernel on `stream` into local [count][5] and all-gathered into
 * gathered [world][count][5] on a side stream the communicator owns, fenced by
 * events -- `stream` is free to run the next steps at once (the reference writes
 * log rows at log-spaced episodes only: utils/wrappers.py:99-110).  local and
 * gathered are caller-owned device buffers that must stay valid until
 * bsb_comm_wait(comm, s), which makes stream `s` wait (on the device) for the
 * latest gather.  As for bsb_sum_episode_stats_many, a handle repeated in `envs`
 * returns BSB_INVALID_ARGUMENT before any reduction or gather is enqueued.
 * Replaces the process pool's result collection of
 * bsuite/baselines/utils/pool.py:28-54.
 */
#define BSB_COMM_ID_BYTES 128
typedef struct bsb_comm bsb_comm;
int32_t bsb_comm_unique_id(uint8_t* id /* [BSB_COMM_ID_BYTES] */);
int32_t bsb_comm_create(const uint8_t* id, int32_t rank, int32_t world,
                        int32_t device, bsb_comm** out);
int32_t bsb_comm_destroy(bsb_comm* comm);
int32_t bsb_comm_world(const bsb_comm* comm, int32_t* rank, int32_t* world);
int32_t bsb_log_point(bsb_comm* comm, bsb_env* const* envs, int32_t count,
                      double* local, double* gathered, void* stream);
/* bsb_log_point over the rows of bsb_sum_setting_stats: local [rows][5],
 * gathered [world][rows][5]. */
int32_t bsb_log_point_settings(bsb_comm* comm, bsb_env* const* envs, int32_t count,
                               double* local, double* gathered, void* stream);
int32_t bsb_comm_wait(bsb_comm* comm, void* stream);

/* Number of kernels this library has launched in this process (bench evidence). */
int64_t bsb_launch_count(void);

/*
 * Interpolating branch of ImageObservation / to_image (utils/wrappers.py:207-219):
 * skimage.transform.resize(plane, (out_rows, out_cols), preserve_range=True)
 * on each [in_rows, in_cols] float32 plane, broadcast over `channels` trailing
 * floats.  skimage (>= 0.19) computes
 *   1. only when out_rows < in_rows or out_cols < in_cols: a Gaussian
 *      anti-aliasing pass per axis (scipy.ndimage.gaussian_filter, mode
 *      'mirror'), rows first, each pass accumulated in float64 and rounded to
 *      float32;
 *   2. scipy.ndimage.zoom(order=1, mode='mirror', grid_mode=True): per output
 *      pixel sum over the 2 x 2 neighbourhood (row-major, from 0.0) of
 *      value * row_weight * col_weight in float64, rounded to float32;
 *   3. a clip to [min, max] of the unfiltered input plane.
 * The plan does not depend on any environment handle.  The caller builds the
 * tables with numpy, with the operations scipy uses, so they are equal by
 * construction (like the deep_sea mapping tables of bsb_config):
 *   row_index / row_weight  [out_rows][2]  mirrored source rows (i0, i1) and
 *                                          weights (w0, w1) of each output row
 *   col_index / col_weight  [out_cols][2]  the same per output column
 *   row_taps                [row_radius + 1] Gaussian taps of the row pass:
 *                                          centre, then distance 1 .. radius
 *                                          (radius 0 / NULL: no pass)
 *   col_taps                [col_radius + 1] the same for the column pass
 * Every *_len is the number of elements of its table.  Tables are HOST
 * pointers; bsb_image_plan_create copies them (synchronously, to `device`).
 */
typedef struct bsb_image_desc {
  int32_t in_rows, in_cols;       /* h, w of every input plane */
  int32_t out_rows, out_cols;     /* H, W of every output image */
  int32_t channels;               /* C: each output pixel is repeated over C consecutive floats */
  int32_t row_radius, col_radius; /* Gaussian radius per axis; 0 = no pass on that axis */
  int32_t reserved0;
  const int32_t* row_index; int64_t row_index_len;
  const double* row_weight; int64_t row_weight_len;
  const int32_t* col_index; int64_t col_index_len;
  const double* col_weight; int64_t col_weight_len;
  const double* row_taps;   int64_t row_taps_len;
  const double* col_taps;   int64_t col_taps_len;
} bsb_image_desc;

typedef struct bsb_image_plan bsb_image_plan; /* opaque handle */

/* device >= 0: CUDA device ordinal; BSB_DEVICE_HOST: explicit host path. */
int32_t bsb_image_plan_create(const bsb_image_desc* desc, int32_t device,
                              bsb_image_plan** out);
int32_t bsb_image_plan_destroy(bsb_image_plan* plan);

/*
 * in: float32 [batch, in_rows, in_cols], out: float32 [batch, out_rows,
 * out_cols, channels], both dense and caller-owned, in the plan's memory space
 * (float32 only: convert a reduced-dtype observation before resizing it).
 * A device plan enqueues one kernel on `stream` and neither synchronises nor
 * allocates, so the call may be captured into a CUDA graph; a host plan is
 * synchronous.  batch 0 does nothing.  A device plan with a Gaussian pass
 * whose planes do not fit the kernel's shared-memory stage (in_rows *
 * in_cols above 6 144 values) filters through scratch memory the plan owns:
 * launches of such a plan must not overlap, so issue them on one stream (or
 * order the streams with events).  Other plans hold read-only tables only
 * and may run concurrently.  NaN values are skipped by the clip's
 * [min, max] (np.nanmin / np.nanmax, as skimage does when a plane holds NaN).
 */
int32_t bsb_to_image(bsb_image_plan* plan, const float* in, int64_t batch,
                     float* out, void* stream);

/*
 * Device memory for observation buffers.  Observations are mostly zero (a
 * deep_sea tile holds at most one 1.0 in 1 024 floats), and memory created
 * with generic compression is compressed by the L2 on its way to DRAM, so
 * kernels that write such tiles move fewer DRAM bytes.  Kernels, copies and
 * the host see ordinary memory holding the values written.
 *
 * bsb_obs_malloc returns `size` bytes on CUDA device `device` (rounded up to
 * the compressible granularity), or NULL with bsb_last_error() set when the
 * device does not exist or memory is exhausted.  It falls back to plain
 * cudaMalloc memory when the device cannot compress, the compressible backing
 * store is used up, or the driver does not grant compression; it never fails
 * where cudaMalloc would succeed.  bsb_obs_free waits for the device, then
 * releases a pointer bsb_obs_malloc returned.  `stream` is unused by both.
 * The signatures are those of torch.cuda.memory.CUDAPluggableAllocator.
 * Host environments (BSB_DEVICE_HOST) use plain host memory.
 *
 * bsb_obs_memory_info: *supported = the device's generic-compression
 * attribute; *compressed_bytes / *plain_bytes = bytes of live bsb_obs_malloc
 * blocks on `device` that were / were not granted compression.
 */
void* bsb_obs_malloc(ptrdiff_t size, int device, void* stream);
void bsb_obs_free(void* ptr, ptrdiff_t size, int device, void* stream);
int32_t bsb_obs_memory_info(int device, int32_t* supported,
                            uint64_t* compressed_bytes, uint64_t* plain_bytes);

#ifdef __cplusplus
}
#endif
#endif /* BSUITE_B200_H_ */
