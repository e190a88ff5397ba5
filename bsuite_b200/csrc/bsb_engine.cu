// bsuite_b200 engine: handle management, kernel dispatch, explicit host path and
// the extern "C" surface declared in include/bsuite_b200.h.
//
// Build: nvcc -gencode arch=compute_90a,code=sm_90a --fmad=false -lineinfo ...
// (--fmad=false: CPython/numpy never contract a*b+c; the float-dynamics
// families must evaluate the reference's expressions operation by operation.)
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <atomic>
#include <chrono>
#if defined(__x86_64__)
#include <immintrin.h>
#endif

#include "bsb_env.h"

using namespace bsb;

namespace bsb {
std::atomic<int64_t> g_launches{0};
namespace { thread_local std::string g_last_error; }
int fail(int code, const std::string& msg) { g_last_error = msg; return code; }
const char* last_error_cstr() { return g_last_error.c_str(); }
}  // namespace bsb

namespace {

InfoNames info_names(int family) {
  switch (family) {
    case BSB_DEEP_SEA: return {2, {"total_bad_episodes", "denoised_return", nullptr, nullptr}};
    case BSB_CATCH: return {1, {"total_regret", nullptr, nullptr, nullptr}};
    case BSB_CARTPOLE: return {2, {"raw_return", "best_episode", nullptr, nullptr}};
    case BSB_CARTPOLE_SWINGUP: return {3, {"raw_return", "total_upright", "best_episode", nullptr}};
    case BSB_MOUNTAIN_CAR: return {1, {"raw_return", nullptr, nullptr, nullptr}};
    case BSB_MEMORY_CHAIN: return {2, {"total_perfect", "total_regret", nullptr, nullptr}};
    case BSB_BANDIT: return {1, {"total_regret", nullptr, nullptr, nullptr}};
    case BSB_UMBRELLA_CHAIN: return {1, {"total_regret", nullptr, nullptr, nullptr}};
    case BSB_DISCOUNTING_CHAIN: return {0, {nullptr, nullptr, nullptr, nullptr}};
    case BSB_MNIST: return {1, {"total_regret", nullptr, nullptr, nullptr}};
  }
  return {0, {nullptr, nullptr, nullptr, nullptr}};
}

}  // namespace

namespace {

struct DeviceGuard {
  int prev; bool on;
  explicit DeviceGuard(int dev) : prev(0), on(dev >= 0) { if (on) { cudaGetDevice(&prev); cudaSetDevice(dev); } }
  ~DeviceGuard() { if (on) cudaSetDevice(prev); }
};

int env_alloc(bsb_env* e, void** out, size_t bytes, bool snapshot) {
  if (bytes == 0) { *out = nullptr; return BSB_OK; }
  void* ptr = nullptr;
  if (e->device >= 0) {
    BSB_CUDA(cudaMalloc(&ptr, bytes));
    BSB_CUDA(cudaMemset(ptr, 0, bytes));
  } else {
    ptr = calloc(1, bytes);
    if (!ptr) return fail(BSB_OUT_OF_MEMORY, "calloc failed");
  }
  e->allocs.push_back(ptr);
  if (snapshot) e->state_blocks.push_back(std::make_pair(ptr, bytes));
  *out = ptr;
  return BSB_OK;
}

int env_upload(bsb_env* e, void* dst, const void* src, size_t bytes) {
  if (bytes == 0) return BSB_OK;
  if (e->device >= 0) { BSB_CUDA(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice)); }
  else memcpy(dst, src, bytes);
  return BSB_OK;
}

template <class T> int env_alloc_t(bsb_env* e, T** out, size_t count, bool snapshot) {
  void* ptr = nullptr;
  int rc = env_alloc(e, &ptr, count * sizeof(T), snapshot);
  *out = static_cast<T*>(ptr);
  return rc;
}

// `two_phase`: a two-phase host step (mailbox_launch; deep_sea and catch only).  `mask`: a masked call, rollout or
// host step (`episodes_left`: the budgets, nullable; `mask_out`: a budgeted host step's mask write-back, nullable;
// `previous`: a budgeted step's previous outputs, nullable; `policy`: a budgeted step's selection rule, nullable;
// `replay`: the rings a recorded step appends to, nullable; `sequence`: the buffers a sequence step appends to,
// nullable; `ensemble`: an ensemble step's heads and values, nullable).
int run(bsb_env* e, const LaunchArgs& args, cudaStream_t stream, const TwoPhaseArgs* two_phase = nullptr,
        const uint8_t* mask = nullptr, int64_t* episodes_left = nullptr, uint8_t* mask_out = nullptr,
        const bsb_outputs* previous = nullptr, const bsb_policy* policy = nullptr, const bsb_replay* replay = nullptr,
        const bsb_sequence* sequence = nullptr, const bsb_ensemble_policy* ensemble = nullptr) {
  DeviceGuard guard(e->device);
  LaunchArgs a = args;
  if (e->device >= 0) {
    cudaStreamCaptureStatus capture = cudaStreamCaptureStatusNone;
    BSB_CUDA(cudaStreamIsCapturing(stream, &capture));
    if (capture != cudaStreamCaptureStatusNone) e->graph_safe = true;
    if (e->graph_safe) a.clock = e->clock;      // a.step0 == e->steps_done, which no longer moves
  }
  if (mask)
    return e->variant->run_masked(e, a, mask, episodes_left, mask_out, previous, policy, replay, sequence, ensemble,
                                  stream);
  return e->variant->run(e, a, stream, two_phase);
}

LaunchArgs make_args(const bsb_env* e, const bsb_outputs* out, const int32_t* actions, int64_t T, int mode) {
  LaunchArgs a;
  memset(&a, 0, sizeof(a));
  a.actions = actions;
  if (out) { a.obs = out->observation; a.reward = out->reward; a.reward_f64 = out->reward_f64; a.discount = out->discount; a.step_type = out->step_type; a.final_obs = out->final_observation; }
  a.T = T; a.step0 = e->steps_done; a.mode = mode;
  const size_t step_bytes = (size_t)e->step_elems * (size_t)e->obs_elem_bytes;
  a.obs_vec_ok = (out && (reinterpret_cast<uintptr_t>(out->observation) % 16 == 0) && (T == 1 || step_bytes % 16 == 0)) ? 1 : 0;
  a.final_vec_ok = (a.final_obs && (reinterpret_cast<uintptr_t>(a.final_obs) % 16 == 0) && (T == 1 || step_bytes % 16 == 0)) ? 1 : 0;
  return a;
}

// The bsb_family of each family and the bsb_obs_dtype of each observation element type.
template <class F> struct FamilyId;
#define BSB_FAMILY_ID(F, id) template <> struct FamilyId<F> { static const int value = id; };
BSB_FAMILY_ID(DeepSea, BSB_DEEP_SEA) BSB_FAMILY_ID(Catch, BSB_CATCH) BSB_FAMILY_ID(Cartpole, BSB_CARTPOLE)
BSB_FAMILY_ID(CartpoleSwingup, BSB_CARTPOLE_SWINGUP) BSB_FAMILY_ID(MountainCar, BSB_MOUNTAIN_CAR)
BSB_FAMILY_ID(MemoryChain, BSB_MEMORY_CHAIN) BSB_FAMILY_ID(Bandit, BSB_BANDIT) BSB_FAMILY_ID(UmbrellaChain, BSB_UMBRELLA_CHAIN)
BSB_FAMILY_ID(DiscountingChain, BSB_DISCOUNTING_CHAIN) BSB_FAMILY_ID(Mnist, BSB_MNIST)
#undef BSB_FAMILY_ID
template <class O> constexpr int obs_dtype_id() {
  return std::is_same<O, float>::value ? BSB_OBS_FLOAT32 : std::is_same<O, Bf16>::value ? BSB_OBS_BFLOAT16 : BSB_OBS_UINT8;
}

#define BSB_ENTRY(F, O, mode, mt, two_phase) \
  {FamilyId<F>::value, obs_dtype_id<O>(), mode, mt, two_phase, &run_variant<Variant<F, O, mode> >, &run_masked<Variant<F, O, mode> >},
const VariantEntry kVariants[] = {BSB_VARIANTS(BSB_ENTRY)};
#undef BSB_ENTRY

// The compiled variant of a family, obs_dtype and mode that runs bit source `rng_kind`, or nullptr.
const VariantEntry* find_variant(int family, int obs_dtype, int mode, int rng_kind) {
  for (const VariantEntry& v : kVariants)
    if (v.family == family && v.obs_dtype == obs_dtype && v.mode == mode && (rng_kind != BSB_RNG_MT19937 || v.mt)) return &v;
  return nullptr;
}

int validate(const bsb_config& c, int64_t batch, int* obs_rows, int* obs_cols, int* n_actions) {
  if (batch <= 0) return fail(BSB_INVALID_ARGUMENT, "batch must be positive");
  if (c.wrapper < 0 || c.wrapper > 2) return fail(BSB_INVALID_ARGUMENT, "unknown wrapper");
  if (c.rng_kind < 0 || c.rng_kind > 1) return fail(BSB_INVALID_ARGUMENT, "unknown rng_kind");
  switch (c.family) {
    case BSB_DEEP_SEA:
      if (c.size < 1 || c.size > 255) return fail(BSB_INVALID_ARGUMENT, "deep_sea size must be in [1, 255]");
      if (!c.table || c.table_bytes != (int64_t)c.size * c.size) return fail(BSB_INVALID_ARGUMENT, "deep_sea needs a uint8 [N*N] action mapping table");
      *obs_rows = c.size; *obs_cols = c.size; *n_actions = 2; break;
    case BSB_CATCH:
      if (c.rows < 2 || c.rows > 255 || c.columns < 1 || c.columns > 255) return fail(BSB_INVALID_ARGUMENT, "catch rows in [2,255], columns in [1,255]");
      *obs_rows = c.rows; *obs_cols = c.columns; *n_actions = 3; break;
    case BSB_CARTPOLE: *obs_rows = 1; *obs_cols = 6; *n_actions = 3; break;
    case BSB_CARTPOLE_SWINGUP: *obs_rows = 1; *obs_cols = 8; *n_actions = 3; break;
    case BSB_MOUNTAIN_CAR:
      if (c.max_steps < 1) return fail(BSB_INVALID_ARGUMENT, "mountain_car max_steps must be >= 1");
      *obs_rows = 1; *obs_cols = 3; *n_actions = 3; break;
    case BSB_MEMORY_CHAIN:
      if (c.num_bits < 1 || c.num_bits > 64) return fail(BSB_UNSUPPORTED, "memory_chain num_bits must be in [1, 64]");
      if (c.memory_length < 1 || c.memory_length >= (1 << 24)) return fail(BSB_INVALID_ARGUMENT, "memory_length must be in [1, 2^24)");
      *obs_rows = 1; *obs_cols = c.num_bits + 2; *n_actions = 2; break;
    case BSB_BANDIT:
      if (c.num_actions < 1) return fail(BSB_INVALID_ARGUMENT, "bandit num_actions must be >= 1");
      if (!c.table || c.table_bytes != (int64_t)c.num_actions * 8) return fail(BSB_INVALID_ARGUMENT, "bandit needs a float64 [num_actions] reward table");
      *obs_rows = 1; *obs_cols = 1; *n_actions = c.num_actions; break;
    case BSB_UMBRELLA_CHAIN:
      if (c.chain_length < 1 || c.chain_length >= (1 << 24)) return fail(BSB_INVALID_ARGUMENT, "chain_length must be in [1, 2^24)");
      if (c.n_distractor < 0 || c.n_distractor > 1533) return fail(BSB_UNSUPPORTED, "n_distractor must be in [0, 1533]");
      *obs_rows = 1; *obs_cols = 3 + c.n_distractor; *n_actions = 2; break;
    case BSB_DISCOUNTING_CHAIN:
      if (!c.table || c.table_bytes != 5 * 8) return fail(BSB_INVALID_ARGUMENT, "discounting_chain needs a float64 [5] reward table");
      *obs_rows = 1; *obs_cols = 2; *n_actions = 5; break;
    case BSB_MNIST:
      if (c.num_data < 1 || c.image_rows < 1 || c.image_cols < 1) return fail(BSB_INVALID_ARGUMENT, "mnist needs num_data, image_rows, image_cols");
      if (c.image_rows > 4096 || c.image_cols > 4096) return fail(BSB_UNSUPPORTED, "mnist image sides must be <= 4096");
      if (!c.table || c.table_bytes != (int64_t)c.num_data * c.image_rows * c.image_cols) return fail(BSB_INVALID_ARGUMENT, "mnist needs an int8 image table");
      if (!c.table2 || c.table2_bytes != c.num_data) return fail(BSB_INVALID_ARGUMENT, "mnist needs a uint8 label table");
      *obs_rows = c.image_rows; *obs_cols = c.image_cols; *n_actions = 10; break;
    default: return fail(BSB_INVALID_ARGUMENT, "unknown family");
  }
  if (c.obs_dtype < BSB_OBS_FLOAT32 || c.obs_dtype > BSB_OBS_UINT8) return fail(BSB_INVALID_ARGUMENT, "unknown obs_dtype");
  if (!find_variant(c.family, c.obs_dtype, NEXT_STEP, BSB_RNG_PHILOX))
    return fail(BSB_UNSUPPORTED, "obs_dtype uint8 is only available for deep_sea and catch, whose observations are 0 / 1");
  if (!find_variant(c.family, c.obs_dtype, NEXT_STEP, c.rng_kind))
    return fail(BSB_UNSUPPORTED, "a bfloat16 or uint8 obs_dtype needs rng_kind BSB_RNG_PHILOX");
  if ((c.flags & BSB_FLAG_SAME_STEP_RESET) && !find_variant(c.family, c.obs_dtype, SAME_STEP, c.rng_kind))
    return fail(BSB_UNSUPPORTED, "BSB_FLAG_SAME_STEP_RESET needs rng_kind BSB_RNG_PHILOX");
  if (c.log_schedule_len < 0 || c.log_schedule_len > 4096) return fail(BSB_INVALID_ARGUMENT, "log_schedule_len must be in [0, 4096]");
  if (c.log_schedule_len > 0) {
    if (!c.log_schedule) return fail(BSB_INVALID_ARGUMENT, "log_schedule_len > 0 needs a log_schedule");
    if (!(c.flags & BSB_FLAG_TRACK_EPISODES)) return fail(BSB_INVALID_ARGUMENT, "a log schedule needs BSB_FLAG_TRACK_EPISODES");
    for (int64_t k = 0; k < c.log_schedule_len; ++k)
      if (c.log_schedule[k] < 1 || (k > 0 && c.log_schedule[k] <= c.log_schedule[k - 1]))
        return fail(BSB_INVALID_ARGUMENT, "log_schedule must be positive and strictly ascending");
  }
  return BSB_OK;
}

bool family_uses_env_rng(const bsb_config& c) {
  switch (c.family) {
    case BSB_DEEP_SEA: return !c.deterministic;
    case BSB_BANDIT: case BSB_DISCOUNTING_CHAIN: return false;
    default: return true;
  }
}
bool family_uses_env_gauss(const bsb_config& c) { return c.family == BSB_DEEP_SEA && !c.deterministic; }

// Device-side alias of a pinned (page-locked, mapped) host pointer, or nullptr for pageable memory.  Queried on
// every call (well under a microsecond): a cached answer could outlive the buffer it described.
void* mapped_device_pointer(bsb_env*, const void* host_ptr) {
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, host_ptr) == cudaSuccess && attr.type == cudaMemoryTypeHost) return attr.devicePointer;
  cudaGetLastError();   // clear the error a pageable pointer may leave behind
  return nullptr;
}


// Host-supplied actions are validated before anything moves (the reference raises IndexError for an arm that does
// not exist: bandit.py:61; catch.py:84).  Device-resident actions cannot be inspected without a synchronise: the
// kernels clamp them and raise env->bad_action_host instead (bsb_invalid_actions).
int check_host_actions(const bsb_env* e, const int32_t* actions, int64_t count) {
  const uint32_t n = (uint32_t)e->p.num_actions;
  for (int64_t k = 0; k < count; ++k)
    if ((uint32_t)actions[k] >= n)
      return fail(BSB_INVALID_ARGUMENT, "action " + std::to_string(actions[k]) + " at index " + std::to_string(k) +
                                            " is outside [0, " + std::to_string(n) + ")");
  return BSB_OK;
}

inline void cpu_relax() {
#if defined(__x86_64__)
  _mm_pause();
#endif
}

// ---- host-driven steps: completion through the mailbox ------------------------------------------------------
int mailbox_open(bsb_env* e) {
  if (e->mailbox) return BSB_OK;
  void* host = nullptr; void* dev = nullptr;
  BSB_CUDA(cudaHostAlloc(&host, sizeof(HostMailbox), cudaHostAllocMapped | cudaHostAllocPortable));
  memset(host, 0, sizeof(HostMailbox));
  BSB_CUDA(cudaHostGetDevicePointer(&dev, host, 0));
  BSB_CUDA(cudaMalloc(reinterpret_cast<void**>(&e->mail), sizeof(DeviceMail)));
  BSB_CUDA(cudaMemset(e->mail, 0, sizeof(DeviceMail)));
  e->mailbox = static_cast<HostMailbox*>(host);
  e->mailbox_dev = static_cast<HostMailbox*>(dev);
  return BSB_OK;
}

// Two-phase host steps pay off where the observation stream is long next to the scalar traffic over PCIe (12 B per
// lane out, 4 B in): deep_sea from N = 16 up (>= 1 KB of observation per lane).  catch (200 B per lane) is bound
// by the 2 MB of scalars per step either way and keeps the single-phase kernel.  The rule counts float32 bytes
// whatever the handle's obs_dtype, so a reduced-dtype handle takes the same path as its float32 twin.
// Only the variants the list compiles two_phase_host_kernel for (deep_sea and catch, next-step) take it.
bool family_obs_from_state(const bsb_env* e) {
  return e->variant->two_phase && (size_t)e->p.obs_numel * sizeof(float) >= 1024;
}

// Device staging of the scalars of host steps: reward | discount | step_type in ONE block, so that a caller who
// keeps its three host arrays back to back (BatchedEnvironment.make_host_buffers does) gets them with a single D2H
// copy; float64 rewards in a block of their own when `f64`.
int alloc_scalar_staging(bsb_env* e, bool f64) {
  const size_t B = (size_t)e->p.batch;
  if (!e->d_reward) {
    BSB_CUDA(cudaMalloc(&e->d_reward, 3 * B * 4));
    e->d_discount = e->d_reward + B;
    e->d_step_type = reinterpret_cast<int32_t*>(e->d_reward + 2 * B);
  }
  if (f64 && !e->d_reward64) BSB_CUDA(cudaMalloc(&e->d_reward64, B * 8));
  return BSB_OK;
}

// True when the caller's reward, discount and step_type arrays lie back to back in one block of 3 * B words.
bool scalars_back_to_back(const bsb_outputs& out, size_t B) {
  return out.reward && out.discount == out.reward + B &&
         reinterpret_cast<char*>(out.step_type) == reinterpret_cast<char*>(out.reward + 2 * B);
}

// Enqueues the step of `actions` into the device-addressable buffers `out`, which signals `ticket` through the
// mailbox.  `mask` (a masked host step; `episodes_left` and `mask_out` nullable): one masked_kernel launch, whose
// observations are written when it signals, so it never takes the two-phase kernel.
int mailbox_launch(bsb_env* e, unsigned long long ticket, const int32_t* actions, const bsb_outputs& out,
                   const uint8_t* mask = nullptr, int64_t* episodes_left = nullptr, uint8_t* mask_out = nullptr) {
  LaunchArgs a = make_args(e, &out, actions, 1, MODE_STEP);
  a.mailbox = e->mailbox_dev; a.mail = e->mail; a.ticket = ticket;
  { static const int timing = getenv("BSB_HOST_TIMING") ? atoi(getenv("BSB_HOST_TIMING")) : 0; a.timing = timing; }
  if (mask) return run(e, a, e->copy_stream, nullptr, mask, episodes_left, mask_out);
  if (!family_obs_from_state(e)) return run(e, a, e->copy_stream);
  { int src = alloc_scalar_staging(e, true); if (src != BSB_OK) return src; }
  TwoPhaseArgs h;
  memset(&h, 0, sizeof(h));
  h.stage.reward = e->d_reward; h.stage.reward_f64 = e->d_reward64; h.stage.discount = e->d_discount; h.stage.step_type = e->d_step_type;
  e->early_inflight = true;
  return run(e, a, e->copy_stream, &h);
}

// Spins on the mailbox until `ticket` is done (the kernel's last CTA stores it after a system-scope fence).
int mailbox_wait(bsb_env* e, unsigned long long ticket) {
  const auto start = std::chrono::steady_clock::now();
  uint32_t spins = 0;
  while (e->mailbox->done < ticket) {
    cpu_relax();
    if ((++spins & 0xfffffu) == 0 && std::chrono::steady_clock::now() - start > std::chrono::seconds(20)) {
      cudaError_t err = cudaStreamSynchronize(e->copy_stream);      // a faulted kernel never signals: surface its error
      if (err != cudaSuccess) return fail(BSB_CUDA_ERROR, std::string("host step: ") + cudaGetErrorString(err));
      if (e->mailbox->done >= ticket) break;
      return fail(BSB_INTERNAL, "host step: the kernel finished without signalling the mailbox");
    }
  }
  std::atomic_thread_fence(std::memory_order_acquire);
  return BSB_OK;
}

// Collects a step issued with BSB_HOST_NO_WAIT: spins until its completion word is in and counts the step.
// Every entry point that enqueues work for this handle or reads its state calls this first.
int finish_awaited(bsb_env* e) {
  if (!e || e->device < 0 || !e->awaiting_ticket) return BSB_OK;
  const unsigned long long ticket = e->awaiting_ticket;
  e->awaiting_ticket = 0;
  int rc = mailbox_wait(e, ticket);
  if (rc != BSB_OK) return rc;
  e->steps_done += 1;
  return BSB_OK;
}

// Two-phase host steps return when the scalars have landed; the observation stores of the latest one may still
// be in flight on the handle's stream.  Anything that leaves that stream (work on a caller's stream, state reads,
// destruction) waits for it here.
int drain_host_steps(bsb_env* e) {
  int rc = finish_awaited(e);
  if (rc != BSB_OK) return rc;
  if (e && e->device >= 0 && e->early_inflight) {
    DeviceGuard guard(e->device);
    e->early_inflight = false;
    BSB_CUDA(cudaStreamSynchronize(e->copy_stream));
  }
  return BSB_OK;
}

void destroy_env(bsb_env* e) {
  drain_host_steps(e);
  DeviceGuard guard(e->device);
  for (size_t k = 0; k < e->allocs.size(); ++k) { if (e->device >= 0) cudaFree(e->allocs[k]); else free(e->allocs[k]); }
  if (e->device >= 0) {
    if (e->h2d_actions) cudaFree(e->h2d_actions);
    if (e->d_reward) cudaFree(e->d_reward);      // also owns d_discount / d_step_type
    if (e->d_reward64) cudaFree(e->d_reward64);
    if (e->d_obs) cudaFree(e->d_obs);
    if (e->d_mask) cudaFree(e->d_mask);
    if (e->copy_stream) cudaStreamDestroy(e->copy_stream);
    if (e->order_event) cudaEventDestroy(e->order_event);
    if (e->fence_event) cudaEventDestroy(e->fence_event);
    if (e->h2d_event) cudaEventDestroy(e->h2d_event);
    if (e->h2d_stream) cudaStreamDestroy(e->h2d_stream);
    if (e->bad_action_host) cudaFreeHost(e->bad_action_host);
    if (e->mailbox) cudaFreeHost(e->mailbox);
    if (e->mail) cudaFree(e->mail);
  }
  delete e;
}

}  // namespace

namespace bsb {
int drain_log_rows(bsb_env* e) { return drain_host_steps(e); }
}  // namespace bsb

__global__ void episode_stat_kernel(const EnvParams p, int field, int64_t calls, const unsigned long long* clock, double* dst) {
  if (clock) calls += (int64_t)*clock;      // graph-safe mode: steps since the switch are counted on the device
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < p.batch) dst[i] = episode_stat(p, i, field, calls);
}

// Sums of the five Logging columns over the lanes of up to kSumManyMax environments in ONE launch (blockIdx.y = row:
// a log point of the 23-experiment sweep is one kernel instead of 23).  A row sums the contiguous lane range
// [first, first + lanes) of a handle whose per-lane arrays have stride `batch`: the whole handle is the range
// (0, batch), setting k of a pack is (k * lanes, lanes).  A job covers `n_settings` consecutive rows; row_start[j] is
// the first row of job j.  Deterministic: a fixed grid of block-strided partial sums, counted from `first`, lands in
// the row's own scratch[block][5]; the block that finishes last adds the partials in block order and re-arms the
// row's ticket.  So a row's order is the one a standalone handle of `lanes` lanes sums in.  (No floating-point
// atomics: the result must not depend on scheduling -- a graph replay and an eager call must agree to the bit.)
constexpr int kSumBlocks = 64, kSumThreads = 256, kSumManyMax = 64;
constexpr int kSumScratch = kSumBlocks * 5 + 1;      // doubles per row: the partials, then the ticket
struct SumJob {
  const double* ep; int64_t batch; int64_t lanes; int64_t calls; const unsigned long long* clock; double* scratch;
  int32_t n_settings;
};
struct SumJobs { SumJob job[kSumManyMax]; int32_t row_start[kSumManyMax]; int32_t count; };
static_assert(sizeof(SumJobs) + sizeof(double*) <= 4096, "kernel parameters must stay within 4 KB");
__global__ void episode_sum_many_kernel(const SumJobs jobs, double* dst) {
  const int row = (int)blockIdx.y;
  int h = 0;
  while (h + 1 < jobs.count && jobs.row_start[h + 1] <= row) ++h;
  const SumJob j = jobs.job[h];
  const int setting = row - jobs.row_start[h];
  const int64_t first = (int64_t)setting * j.lanes;
  double* scratch = j.scratch + (int64_t)setting * kSumScratch;
  EnvParams p;
  p.ep = const_cast<double*>(j.ep); p.batch = j.batch;
  int64_t calls = j.calls;
  if (j.clock) calls += (int64_t)*j.clock;      // graph-safe mode: steps since the switch are counted on the device
  __shared__ double partial[5][kSumThreads / 32];
  __shared__ bool is_last;
  double v[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < j.lanes; i += (int64_t)gridDim.x * blockDim.x)
#pragma unroll
    for (int f = 0; f < 5; ++f) v[f] += episode_stat(p, first + i, f, calls);
#pragma unroll
  for (int f = 0; f < 5; ++f)
    for (int o = 16; o > 0; o >>= 1) v[f] += __shfl_down_sync(0xffffffffu, v[f], o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) for (int f = 0; f < 5; ++f) partial[f][warp] = v[f];
  __syncthreads();
  // blocks that own no lanes of this row contribute exact zeros, so the block-order sum below equals the one a grid
  // of min(blocks, ceil(lanes / threads)) blocks forms (bsb_sum_episode_stats launches that many)
  if (threadIdx.x < 5) {
    double s = 0.0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += partial[threadIdx.x][w];
    scratch[blockIdx.x * 5 + threadIdx.x] = s;
    __threadfence();
  }
  __syncthreads();
  unsigned long long* ticket = reinterpret_cast<unsigned long long*>(scratch + kSumBlocks * 5);
  if (threadIdx.x == 0) is_last = atomicAdd(ticket, 1ull) == (unsigned long long)gridDim.x - 1ull;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (threadIdx.x < 5) {
    double s = 0.0;
    for (unsigned b = 0; b < gridDim.x; ++b) s += __ldcg(scratch + b * 5 + threadIdx.x);
    dst[blockIdx.y * 5 + threadIdx.x] = s;
  }
  if (threadIdx.x == 0) *ticket = 0ull;
}

// ============================ extern "C" ====================================
extern "C" {

int32_t bsb_abi_version(void) { return BSB_ABI_VERSION; }
const char* bsb_last_error(void) { return bsb::last_error_cstr(); }
int64_t bsb_launch_count(void) { return g_launches.load(); }

// Observation elements of a ragged pack's blocks are 128-byte aligned (32 float32 elements).
static int64_t align_block(int64_t elems) { return (elems + 31) / 32 * 32; }

// bsb_create, and bsb_create_packed / bsb_create_ragged with `n_settings` > 0 (`config` is then configs[0], the
// validated settings are `configs` with their `seeds`; `batch` = n_settings * lanes_per_setting).
static int32_t create_env(const bsb_config* config, int64_t batch, int32_t device, uint64_t seed, uint64_t lane_offset,
                          bsb_env** out, const bsb_config* configs = nullptr, const uint64_t* seeds = nullptr,
                          int32_t n_settings = 0, bool ragged = false) {
  if (!config || !out) return fail(BSB_INVALID_ARGUMENT, "null argument");
  *out = nullptr;
  const bsb_config& c = *config;
  int obs_rows = 0, obs_cols = 0, n_actions = 0;
  int rc = validate(c, batch, &obs_rows, &obs_cols, &n_actions);
  if (rc != BSB_OK) return rc;
  const int mode = ragged ? RAGGED : n_settings > 0 ? PACKED : (c.flags & BSB_FLAG_SAME_STEP_RESET) ? SAME_STEP : NEXT_STEP;
  const VariantEntry* variant = find_variant(c.family, c.obs_dtype, mode, c.rng_kind);
  if (!variant) return fail(BSB_INTERNAL, "no compiled kernel variant for this family, obs_dtype, mode and rng_kind");
  if (device >= 0) {
    int count = 0;
    cudaError_t err = cudaGetDeviceCount(&count);
    if (err != cudaSuccess || count <= 0)
      return fail(BSB_CUDA_ERROR, std::string("no CUDA device available (") + cudaGetErrorString(err) +
                                      "); this engine has no implicit CPU fallback -- pass device=BSB_DEVICE_HOST explicitly for the host path");
    if (device >= count) return fail(BSB_INVALID_ARGUMENT, "device ordinal out of range");
  } else if (device != BSB_DEVICE_HOST) {
    return fail(BSB_INVALID_ARGUMENT, "device must be >= 0 or BSB_DEVICE_HOST");
  }

  bsb_env* e = new bsb_env();
  memset(&e->p, 0, sizeof(e->p));
  e->device = device; e->steps_done = 0;
  e->obs_dtype = c.obs_dtype; e->obs_elem_bytes = c.obs_dtype == BSB_OBS_BFLOAT16 ? 2 : c.obs_dtype == BSB_OBS_UINT8 ? 1 : 4;
  e->same_step = (c.flags & BSB_FLAG_SAME_STEP_RESET) != 0;
  e->variant = variant;
  e->packed = n_settings > 0; e->n_settings = n_settings > 0 ? n_settings : 1;
  e->lanes_per_setting = n_settings > 0 ? batch / n_settings : batch;
  e->ragged = ragged;
  {  // the observation blocks: one per setting, back to back (ragged packs: 128-byte aligned, each of its own shape)
    const int32_t n = e->n_settings;
    int64_t at = 0;
    for (int32_t k = 0; k < n; ++k) {
      int rows = obs_rows, cols = obs_cols, unused = 0;
      if (ragged) validate(configs[k], batch, &rows, &cols, &unused);
      e->obs_offset.push_back(at);
      e->obs_rows.push_back(rows); e->obs_cols.push_back(cols);
      at += e->lanes_per_setting * (int64_t)rows * cols;
      if (ragged) at = align_block(at);
    }
    e->step_elems = at;
  }
  e->graph_safe = false; e->clock = nullptr; e->sum_scratch = nullptr; e->names = info_names(c.family);
  e->work_counter = nullptr; e->work_base = 0;
  e->num_sms = 132;
  if (device >= 0) { int n = 0; if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, device) == cudaSuccess && n > 0) e->num_sms = n; }
  e->order_event = nullptr; e->fence_event = nullptr; e->bad_action_host = nullptr; e->bad_action_dev = nullptr;
  e->mailbox = nullptr; e->mailbox_dev = nullptr; e->mail = nullptr; e->next_ticket = 0; e->awaiting_ticket = 0;
  e->h2d_stream = nullptr; e->h2d_event = nullptr;
  e->early_inflight = false;
  e->h2d_actions = nullptr; e->d_reward = nullptr; e->d_reward64 = nullptr; e->d_discount = nullptr; e->d_step_type = nullptr; e->d_obs = nullptr;
  e->d_mask = nullptr;
  e->copy_stream = nullptr;
  DeviceGuard guard(device);

  EnvParams& p = e->p;
  p.family = c.family; p.wrapper = c.wrapper; p.rng_kind = c.rng_kind; p.flags = c.flags;
  p.size = c.size; p.deterministic = c.deterministic; p.rows = c.rows; p.columns = c.columns;
  p.memory_length = c.memory_length; p.num_bits = c.num_bits; p.chain_length = c.chain_length; p.n_distractor = c.n_distractor;
  p.num_actions = n_actions; p.max_steps = c.max_steps; p.num_data = c.num_data; p.image_numel = c.family == BSB_MNIST ? c.image_rows * c.image_cols : 0;
  p.obs_rows = obs_rows; p.obs_cols = obs_cols; p.obs_numel = obs_rows * obs_cols; p.n_info = e->names.n;
  if (ragged) {      // the launch plan sizes the stages for the largest observation; each chunk uses its setting's
    for (int32_t k = 0; k < n_settings; ++k) p.obs_numel = std::max(p.obs_numel, e->obs_rows[k] * e->obs_cols[k]);
  }
  p.batch = batch; p.seed = seed; p.lane_offset = lane_offset;
  if (c.family == BSB_DEEP_SEA) { p.move_cost_step = c.unscaled_move_cost / (double)c.size; p.inv_size = 1.0 / (double)c.size; }
  p.height_threshold = c.height_threshold; p.x_threshold = c.x_threshold; p.timescale = c.timescale; p.max_time = c.max_time;
  p.init_range = c.init_range; p.theta_dot_threshold = c.theta_dot_threshold; p.x_reward_threshold = c.x_reward_threshold;
  p.move_cost = c.move_cost; p.noise_scale = c.noise_scale; p.reward_scale = c.reward_scale;
  {  // cartpole.py:106-112 and the locals of step_cartpole (:40-47)
    const double mass_cart = 1.0, mass_pole = 0.1, length = 0.5;
    p.cp_force_mag = 10.0; p.cp_gravity = 9.8; p.cp_length = length; p.cp_mass_pole = mass_pole;
    p.cp_pl = mass_pole * length; p.cp_mass_total = mass_cart + mass_pole;
    p.cp_four_thirds = 4.0 / 3.0; p.cp_two_pi = 2.0 * 3.141592653589793;
  }

#define BSB_TRY(expr) do { rc = (expr); if (rc != BSB_OK) { destroy_env(e); return rc; } } while (0)
  const size_t B = (size_t)batch;
  // tables
  std::vector<int64_t> mapping_offset(n_settings > 0 ? (size_t)n_settings : 1, 0);
  if (c.family == BSB_DEEP_SEA) {
    // a ragged pack stacks its settings' mapping bits, setting k from word mapping_offset[k]
    std::vector<uint32_t> bits;
    for (int32_t k = 0; k < (ragged ? n_settings : 1); ++k) {
      const bsb_config& ck = ragged ? configs[k] : c;
      const int cells = ck.size * ck.size;
      mapping_offset[(size_t)k] = (int64_t)bits.size();
      bits.resize(bits.size() + (size_t)(cells + 31) / 32, 0u);
      uint32_t* word = bits.data() + mapping_offset[(size_t)k];
      const uint8_t* m = static_cast<const uint8_t*>(ck.table);
      for (int j = 0; j < cells; ++j) if (m[j]) word[(size_t)j >> 5] |= 1u << (j & 31);
    }
    uint32_t* d = nullptr;
    BSB_TRY(env_alloc_t(e, &d, bits.size(), false));
    BSB_TRY(env_upload(e, d, bits.data(), bits.size() * 4));
    p.mapping_bits = d;
  } else if (c.family == BSB_BANDIT || c.family == BSB_DISCOUNTING_CHAIN) {
    // a packed handle stacks its settings' tables (all of one size), setting k at k * table_bytes / 8
    const size_t tables = e->packed ? (size_t)n_settings : 1;
    double* d = nullptr;
    BSB_TRY(env_alloc_t(e, &d, tables * (size_t)c.table_bytes / 8, false));
    for (size_t k = 0; k < tables; ++k)
      BSB_TRY(env_upload(e, d + k * (size_t)c.table_bytes / 8, e->packed ? configs[k].table : c.table, (size_t)c.table_bytes));
    p.reward_table = d;
  } else if (c.family == BSB_MNIST) {
    int8_t* d = nullptr; uint8_t* l = nullptr;
    BSB_TRY(env_alloc_t(e, &d, (size_t)c.table_bytes, false));
    BSB_TRY(env_upload(e, d, c.table, (size_t)c.table_bytes));
    BSB_TRY(env_alloc_t(e, &l, (size_t)c.table2_bytes, false));
    BSB_TRY(env_upload(e, l, c.table2, (size_t)c.table2_bytes));
    p.images = d; p.labels = l;
  }
  if (device >= 0) {
    BSB_TRY(env_alloc_t(e, &e->work_counter, 1, false));
    BSB_TRY(env_alloc_t(e, &e->clock, CLOCK_WORDS, false));
    // every setting's own partials and ticket, so the rows of one per-setting launch never share them
    BSB_TRY(env_alloc_t(e, &e->sum_scratch, (size_t)e->n_settings * kSumScratch, false));
    void* flag = nullptr; void* flag_dev = nullptr;
    if (cudaHostAlloc(&flag, sizeof(int32_t), cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess ||
        cudaHostGetDevicePointer(&flag_dev, flag, 0) != cudaSuccess) {
      destroy_env(e); return fail(BSB_OUT_OF_MEMORY, "pinned allocation for the invalid-action flag failed");
    }
    e->bad_action_host = static_cast<int32_t*>(flag); *e->bad_action_host = 0;
    e->bad_action_dev = static_cast<int32_t*>(flag_dev);
  } else {
    e->bad_action_flag = 0;
    e->bad_action_host = &e->bad_action_flag;
  }
  // lane state
  BSB_TRY(env_alloc_t(e, &p.st_word, B, true));
  if (c.family == BSB_MEMORY_CHAIN) BSB_TRY(env_alloc_t(e, &p.st_ctx, B, true));
  if (c.family == BSB_CARTPOLE || c.family == BSB_CARTPOLE_SWINGUP) BSB_TRY(env_alloc_t(e, &p.st_f64, 6 * B, true));
  if (c.family == BSB_MOUNTAIN_CAR) BSB_TRY(env_alloc_t(e, &p.st_f64, 2 * B, true));
  BSB_TRY(env_alloc_t(e, &p.info, (size_t)BSB_MAX_INFO * B, true));
  // same-step handles: a sixth column, the marker that restarts episode_len / episode_return (lane_step)
  if (c.flags & BSB_FLAG_TRACK_EPISODES) BSB_TRY(env_alloc_t(e, &p.ep, (e->same_step ? 6 : 5) * B, true));
  if (c.log_schedule_len > 0) {      // per-lane rows at the Logging wrapper's log-spaced episodes (wrappers.py:140-147)
    int64_t* sched = nullptr;
    BSB_TRY(env_alloc_t(e, &sched, (size_t)c.log_schedule_len, false));
    BSB_TRY(env_upload(e, sched, c.log_schedule, (size_t)c.log_schedule_len * sizeof(int64_t)));
    p.log_sched = sched; p.n_log_points = (int32_t)c.log_schedule_len;
    BSB_TRY(env_alloc_t(e, &p.log_rows, (size_t)c.log_schedule_len * (size_t)(5 + e->names.n) * B, true));
    BSB_TRY(env_alloc_t(e, &p.log_next, B, true));
  }
  // RNG state
  const bool env_rng = family_uses_env_rng(c);
  const bool noise = c.wrapper == BSB_WRAP_REWARD_NOISE;
  if (env_rng) {
    BSB_TRY(env_alloc_t(e, &p.rng_pos, B, true));
    if (family_uses_env_gauss(c)) BSB_TRY(env_alloc_t(e, &p.rng_gauss, B, true));
  }
  if (noise) {
    BSB_TRY(env_alloc_t(e, &p.wrng_pos, B, true));
    BSB_TRY(env_alloc_t(e, &p.wrng_gauss, B, true));
  }
  if (c.rng_kind == BSB_RNG_MT19937 && (env_rng || noise)) {
    // numpy.random.RandomState(seed + global lane); the wrapper's RandomState is
    // seeded with the SAME integer as the environment's (wrappers.py:267).
    std::vector<uint32_t> keys(624 * B);
    std::vector<int32_t> idx(B, 624);
    for (size_t i = 0; i < B; ++i) mt19937_seed_host(keys.data() + i, (int64_t)B, (uint32_t)(seed + lane_offset + i));
    if (env_rng) {
      BSB_TRY(env_alloc_t(e, &p.mt_key, 624 * B, true)); BSB_TRY(env_upload(e, p.mt_key, keys.data(), keys.size() * 4));
      BSB_TRY(env_alloc_t(e, &p.mt_idx, B, true)); BSB_TRY(env_upload(e, p.mt_idx, idx.data(), B * 4));
    }
    if (noise) {
      BSB_TRY(env_alloc_t(e, &p.wmt_key, 624 * B, true)); BSB_TRY(env_upload(e, p.wmt_key, keys.data(), keys.size() * 4));
      BSB_TRY(env_alloc_t(e, &p.wmt_idx, B, true)); BSB_TRY(env_upload(e, p.wmt_idx, idx.data(), B * 4));
    }
  }
  if (ragged) {         // the per-setting values and observation blocks of a ragged pack (ragged_setting_params)
    std::vector<char> blob(sizeof(RaggedTable) + (size_t)n_settings * sizeof(RaggedSetting), 0);
    RaggedTable* t = reinterpret_cast<RaggedTable*>(blob.data());
    t->pack.lanes_per_setting = e->lanes_per_setting; t->pack.n_settings = n_settings;
    t->step_elems = e->step_elems;
    t->mapping_bits = c.family == BSB_DEEP_SEA ? p.mapping_bits : nullptr;
    RaggedSetting* s = reinterpret_cast<RaggedSetting*>(t + 1);
    for (int32_t k = 0; k < n_settings; ++k) {
      const bsb_config& ck = configs[k];
      const int32_t K = e->obs_rows[(size_t)k] * e->obs_cols[(size_t)k];
      s[k].seed = seeds[k];
      s[k].lane_shift = (int64_t)k * e->lanes_per_setting;
      s[k].obs_offset = e->obs_offset[(size_t)k];
      s[k].mapping_offset = mapping_offset[(size_t)k];
      s[k].size = ck.size;
      if (c.family == BSB_DEEP_SEA) { s[k].inv_size = 1.0 / (double)ck.size; s[k].move_cost_step = ck.unscaled_move_cost / (double)ck.size; }
      s[k].num_bits = ck.num_bits; s[k].n_distractor = ck.n_distractor; s[k].obs_numel = K;
      s[k].memory_length = ck.memory_length; s[k].chain_length = ck.chain_length;
      s[k].group_lanes = tile_group_lanes((size_t)K * sizeof(float));      // deep_sea: lanes per bulk store
      e->group_lanes.push_back(c.family == BSB_DEEP_SEA ? s[k].group_lanes : 0);
    }
    void* d = nullptr;
    BSB_TRY(env_alloc(e, &d, blob.size(), false));
    BSB_TRY(env_upload(e, d, blob.data(), blob.size()));
    p.pack = static_cast<const PackTable*>(d);
  } else if (e->packed) {      // the per-setting values every lane of a packed handle picks up (pack_lane_params)
    std::vector<char> blob(sizeof(PackTable) + (size_t)n_settings * sizeof(PackSetting));
    PackTable* t = reinterpret_cast<PackTable*>(blob.data());
    t->lanes_per_setting = e->lanes_per_setting; t->n_settings = n_settings;
    PackSetting* s = reinterpret_cast<PackSetting*>(t + 1);
    for (int32_t k = 0; k < n_settings; ++k) {
      const bsb_config& ck = configs[k];
      s[k].seed = seeds[k];
      s[k].table_offset = p.reward_table ? (int64_t)k * (c.table_bytes / 8) : 0;
      s[k].height_threshold = ck.height_threshold; s[k].x_reward_threshold = ck.x_reward_threshold;
      s[k].noise_scale = ck.noise_scale; s[k].reward_scale = ck.reward_scale;
      s[k].memory_length = ck.memory_length; s[k].chain_length = ck.chain_length;
    }
    void* d = nullptr;
    BSB_TRY(env_alloc(e, &d, blob.size(), false));
    BSB_TRY(env_upload(e, d, blob.data(), blob.size()));
    p.pack = static_cast<const PackTable*>(d);
  }
  // constructor: _reset_next_step = True and the constructor's RNG draws
  LaunchArgs a = make_args(e, nullptr, nullptr, 0, MODE_INIT);
  BSB_TRY(run(e, a, nullptr));
  if (device >= 0) {
    cudaError_t err = cudaDeviceSynchronize();
    if (err != cudaSuccess) { destroy_env(e); return fail(BSB_CUDA_ERROR, std::string("init kernel: ") + cudaGetErrorString(err)); }
  }
#undef BSB_TRY
  *out = e;
  return BSB_OK;
}

int32_t bsb_create(const bsb_config* config, int64_t batch, int32_t device, uint64_t seed, uint64_t lane_offset, bsb_env** out) {
  return create_env(config, batch, device, seed, lane_offset, out);
}

// The first field in which two settings of a packed handle differ although they may not (nullptr: none).  Allowed
// to differ: the seed (seeds[]), the contents of `table` (bandit / discounting_chain reward tables), memory_length,
// chain_length, height_threshold, x_reward_threshold, noise_scale, reward_scale.  The settings of a ragged pack
// (`ragged`) may also differ in size with its deep_sea mapping table, num_bits and n_distractor.
static const char* packed_mismatch(const bsb_config& a, const bsb_config& b, bool ragged = false) {
#define BSB_SAME(field) if (memcmp(&a.field, &b.field, sizeof(a.field)) != 0) return #field;
  BSB_SAME(family) BSB_SAME(wrapper) BSB_SAME(rng_kind) BSB_SAME(flags)
  if (!ragged) { BSB_SAME(size) }
  BSB_SAME(deterministic) BSB_SAME(rows) BSB_SAME(columns)
  if (!ragged) { BSB_SAME(num_bits) BSB_SAME(n_distractor) }
  BSB_SAME(num_actions) BSB_SAME(max_steps)
  BSB_SAME(num_data) BSB_SAME(image_rows) BSB_SAME(image_cols) BSB_SAME(obs_dtype) BSB_SAME(unscaled_move_cost)
  BSB_SAME(x_threshold) BSB_SAME(timescale) BSB_SAME(max_time) BSB_SAME(init_range) BSB_SAME(theta_dot_threshold)
  BSB_SAME(move_cost)
  if (!ragged || a.family != BSB_DEEP_SEA) { BSB_SAME(table_bytes) }
  BSB_SAME(table2_bytes) BSB_SAME(log_schedule_len)
#undef BSB_SAME
  if (a.family == BSB_MNIST && a.table_bytes == b.table_bytes && a.table != b.table &&
      (!a.table || !b.table || memcmp(a.table, b.table, (size_t)a.table_bytes) != 0)) return "table";
  if (a.table2_bytes == b.table2_bytes && a.table2 != b.table2 &&
      (!a.table2 || !b.table2 || memcmp(a.table2, b.table2, (size_t)a.table2_bytes) != 0)) return "table2";
  if (a.log_schedule_len == b.log_schedule_len && a.log_schedule != b.log_schedule && a.log_schedule_len > 0 &&
      (!a.log_schedule || !b.log_schedule ||
       memcmp(a.log_schedule, b.log_schedule, (size_t)a.log_schedule_len * sizeof(int64_t)) != 0)) return "log_schedule";
  return nullptr;
}

int32_t bsb_create_packed(const bsb_config* configs, int32_t n_settings, int64_t lanes_per_setting, int32_t device,
                          const uint64_t* seeds, uint64_t lane_offset, bsb_env** out) {
  if (!configs || !seeds || !out) return fail(BSB_INVALID_ARGUMENT, "null argument");
  *out = nullptr;
  if (n_settings < 1 || n_settings > BSB_MAX_PACKED_SETTINGS)
    return fail(BSB_INVALID_ARGUMENT, "n_settings must be in [1, " + std::to_string(BSB_MAX_PACKED_SETTINGS) + "]");
  if (lanes_per_setting < 1 || lanes_per_setting > INT64_MAX / n_settings)
    return fail(BSB_INVALID_ARGUMENT, "lanes_per_setting must be positive (and n_settings * lanes_per_setting an int64)");
  for (int32_t k = 0; k < n_settings; ++k) {
    int rows = 0, cols = 0, n_actions = 0;
    const int rc = validate(configs[k], lanes_per_setting, &rows, &cols, &n_actions);
    if (rc != BSB_OK) return fail(rc, "setting " + std::to_string(k) + ": " + last_error_cstr());
  }
  const bsb_config& c = configs[0];
  if (!find_variant(c.family, BSB_OBS_FLOAT32, PACKED, BSB_RNG_PHILOX))
    return fail(BSB_UNSUPPORTED, "deep_sea has no packed kernel (its settings differ in size)");
  if (!find_variant(c.family, BSB_OBS_FLOAT32, PACKED, c.rng_kind)) return fail(BSB_UNSUPPORTED, "packed handles need rng_kind BSB_RNG_PHILOX");
  if (!find_variant(c.family, c.obs_dtype, PACKED, c.rng_kind)) return fail(BSB_UNSUPPORTED, "packed handles write float32 observations only");
  if (c.flags & BSB_FLAG_SAME_STEP_RESET) return fail(BSB_UNSUPPORTED, "packed handles do not take BSB_FLAG_SAME_STEP_RESET");
  for (int32_t k = 1; k < n_settings; ++k)
    if (const char* field = packed_mismatch(c, configs[k]))
      return fail(BSB_UNSUPPORTED, std::string("settings 0 and ") + std::to_string(k) + " differ in `" + field +
                                       "`, which the settings of a packed handle must share");
  return create_env(&c, (int64_t)n_settings * lanes_per_setting, device, seeds[0], lane_offset, out, configs, seeds,
                    n_settings);
}

int32_t bsb_packed_layout(const bsb_env* env, int32_t* n_settings, int64_t* lanes_per_setting) {
  if (!env || !n_settings || !lanes_per_setting) return fail(BSB_INVALID_ARGUMENT, "null argument");
  *n_settings = env->n_settings; *lanes_per_setting = env->lanes_per_setting;
  return BSB_OK;
}

int32_t bsb_create_ragged(const bsb_config* configs, int32_t n_settings, int64_t lanes_per_setting, int32_t device,
                          const uint64_t* seeds, uint64_t lane_offset, bsb_env** out) {
  if (!configs || !seeds || !out) return fail(BSB_INVALID_ARGUMENT, "null argument");
  *out = nullptr;
  if (n_settings < 1 || n_settings > BSB_MAX_PACKED_SETTINGS)
    return fail(BSB_INVALID_ARGUMENT, "n_settings must be in [1, " + std::to_string(BSB_MAX_PACKED_SETTINGS) + "]");
  if (lanes_per_setting < 1 || lanes_per_setting > INT64_MAX / n_settings)
    return fail(BSB_INVALID_ARGUMENT, "lanes_per_setting must be positive (and n_settings * lanes_per_setting an int64)");
  for (int32_t k = 0; k < n_settings; ++k) {
    int rows = 0, cols = 0, n_actions = 0;
    const int rc = validate(configs[k], lanes_per_setting, &rows, &cols, &n_actions);
    if (rc != BSB_OK) return fail(rc, "setting " + std::to_string(k) + ": " + last_error_cstr());
  }
  const bsb_config& c = configs[0];
  if (!find_variant(c.family, BSB_OBS_FLOAT32, RAGGED, BSB_RNG_PHILOX))
    return fail(BSB_UNSUPPORTED, "`family`: ragged packs hold deep_sea, memory_chain or umbrella_chain; the settings of "
                                 "other families share one observation shape: use bsb_create_packed");
  for (int32_t k = 0; k < n_settings; ++k) {
    const bsb_config& ck = configs[k];
    const char* field = ck.rng_kind != BSB_RNG_PHILOX ? "rng_kind` (ragged packs need BSB_RNG_PHILOX"
                        : ck.obs_dtype != BSB_OBS_FLOAT32 ? "obs_dtype` (ragged packs write float32 observations"
                        : (ck.flags & BSB_FLAG_SAME_STEP_RESET) ? "flags` (ragged packs do not take BSB_FLAG_SAME_STEP_RESET"
                        : ck.wrapper != BSB_WRAP_NONE ? "wrapper` (ragged packs take no reward wrapper"
                        : nullptr;
    if (field) return fail(BSB_UNSUPPORTED, "setting " + std::to_string(k) + ": `" + field + ")");
  }
  for (int32_t k = 1; k < n_settings; ++k)
    if (const char* field = packed_mismatch(c, configs[k], true))
      return fail(BSB_UNSUPPORTED, std::string("settings 0 and ") + std::to_string(k) + " differ in `" + field +
                                       "`, which the settings of a ragged pack must share");
  return create_env(&c, (int64_t)n_settings * lanes_per_setting, device, seeds[0], lane_offset, out, configs, seeds,
                    n_settings, true);
}

int32_t bsb_ragged_layout(const bsb_env* env, int64_t* offsets, int32_t* rows, int32_t* cols, int64_t* step_elems) {
  if (!env || !offsets || !rows || !cols || !step_elems) return fail(BSB_INVALID_ARGUMENT, "null argument");
  for (int32_t k = 0; k < env->n_settings; ++k) {
    offsets[k] = env->obs_offset[(size_t)k]; rows[k] = env->obs_rows[(size_t)k]; cols[k] = env->obs_cols[(size_t)k];
  }
  *step_elems = env->step_elems;
  return BSB_OK;
}

int32_t bsb_destroy(bsb_env* env) { if (env) destroy_env(env); return BSB_OK; }

static int refuse_ragged(const bsb_env* env) {
  if (env->ragged) return fail(BSB_UNSUPPORTED, "the settings of a ragged pack differ in observation shape: read them with bsb_ragged_layout");
  return BSB_OK;
}
int32_t bsb_obs_numel(const bsb_env* env, int64_t* numel) {
  if (!env || !numel) return fail(BSB_INVALID_ARGUMENT, "null argument");
  { int rc = refuse_ragged(env); if (rc != BSB_OK) return rc; }
  *numel = env->p.obs_numel; return BSB_OK;
}
int32_t bsb_obs_shape(const bsb_env* env, int32_t* rows, int32_t* cols) {
  if (!env || !rows || !cols) return fail(BSB_INVALID_ARGUMENT, "null argument");
  { int rc = refuse_ragged(env); if (rc != BSB_OK) return rc; }
  *rows = env->p.obs_rows; *cols = env->p.obs_cols; return BSB_OK;
}
int32_t bsb_num_actions(const bsb_env* env, int32_t* n) {
  if (!env || !n) return fail(BSB_INVALID_ARGUMENT, "null argument");
  *n = env->p.num_actions; return BSB_OK;
}
int32_t bsb_batch(const bsb_env* env, int64_t* batch) {
  if (!env || !batch) return fail(BSB_INVALID_ARGUMENT, "null argument");
  *batch = env->p.batch; return BSB_OK;
}
// Host view of the step counter.  In graph-safe mode the count lives on the device (graph replays advance it
// without the host seeing them): wait for the device and read it back.
static int current_steps(const bsb_env* env, int64_t* steps) {
  *steps = env->steps_done;
  if (env->graph_safe) {
    DeviceGuard guard(env->device);
    unsigned long long since = 0;
    BSB_CUDA(cudaDeviceSynchronize());
    BSB_CUDA(cudaMemcpy(&since, env->clock, sizeof(since), cudaMemcpyDeviceToHost));
    *steps += (int64_t)since;
  }
  return BSB_OK;
}
static void advance_steps(bsb_env* env, int64_t n) { if (!env->graph_safe) env->steps_done += n; }

int32_t bsb_steps_done(const bsb_env* env, int64_t* steps) {
  if (!env || !steps) return fail(BSB_INVALID_ARGUMENT, "null argument");
  int rc = current_steps(env, steps);
  if (rc == BSB_OK && env->awaiting_ticket) *steps += 1;      // a BSB_HOST_NO_WAIT step has been issued: it counts
  return rc;
}

// bsb_outputs.final_observation is for same-step handles only.
static int check_final_observation(const bsb_env* env, const bsb_outputs* out) {
  if (out->final_observation && !env->same_step)
    return fail(BSB_INVALID_ARGUMENT, "final_observation needs a handle created with BSB_FLAG_SAME_STEP_RESET");
  return BSB_OK;
}

int32_t bsb_reset(bsb_env* env, const bsb_outputs* out, void* stream) {
  if (!env || !out || !out->observation) return fail(BSB_INVALID_ARGUMENT, "bsb_reset needs outputs with an observation buffer");
  { int crc = check_final_observation(env, out); if (crc != BSB_OK) return crc; }
  { int frc = drain_host_steps(env); if (frc != BSB_OK) return frc; }
  LaunchArgs a = make_args(env, out, nullptr, 1, MODE_RESET);
  int rc = run(env, a, static_cast<cudaStream_t>(stream));
  if (rc == BSB_OK) advance_steps(env, 1);
  return rc;
}

int32_t bsb_step(bsb_env* env, const int32_t* actions, const bsb_outputs* out, void* stream) {
  if (!env || !actions || !out || !out->observation) return fail(BSB_INVALID_ARGUMENT, "bsb_step needs actions and outputs with an observation buffer");
  { int crc = check_final_observation(env, out); if (crc != BSB_OK) return crc; }
  { int frc = drain_host_steps(env); if (frc != BSB_OK) return frc; }
  if (env->device < 0) { int vrc = check_host_actions(env, actions, env->p.batch); if (vrc != BSB_OK) return vrc; }
  LaunchArgs a = make_args(env, out, actions, 1, MODE_STEP);
  int rc = run(env, a, static_cast<cudaStream_t>(stream));
  if (rc == BSB_OK) advance_steps(env, 1);
  return rc;
}

// bsb_reset_masked / bsb_step_masked / bsb_rollout_masked / bsb_step_host_masked: lane i makes the calls only where
// mask[i] != 0 (run_masked), a rollout's or host step's lanes only while their budgets last.  Host handles validate
// the actions of masked-in lanes only, at every step of a rollout (a host step: of lanes with budget left): an
// inactive lane's action is never read.  `mask_out`: a budgeted host step's write-back, or a budgeted step's mask;
// `previous`: a budgeted step's previous outputs; `policy`: the rule that picks a budgeted step's actions; `replay`:
// the rings a recorded step appends to; `sequence`: the buffers a sequence step appends to; `ensemble`: an ensemble
// step's heads and values (run_masked).
static int masked_call(bsb_env* env, const int32_t* actions, const uint8_t* mask, const bsb_outputs* out, void* stream,
                       int mode, int64_t T = 1, bool rollout = false, uint64_t action_seed = 0,
                       int32_t* actions_out = nullptr, int64_t* episodes_left = nullptr, uint8_t* mask_out = nullptr,
                       const bsb_outputs* previous = nullptr, const bsb_policy* policy = nullptr,
                       const bsb_replay* replay = nullptr, const bsb_sequence* sequence = nullptr,
                       const bsb_ensemble_policy* ensemble = nullptr) {
  { int crc = check_final_observation(env, out); if (crc != BSB_OK) return crc; }
  { int frc = drain_host_steps(env); if (frc != BSB_OK) return frc; }
  if (env->device < 0 && mode == MODE_STEP && actions) {
    const uint32_t n = (uint32_t)env->p.num_actions;
    const int64_t B = env->p.batch;
    for (int64_t t = 0; t < T; ++t)
      for (int64_t k = 0; k < B; ++k)
        if (mask[k] && (rollout || !episodes_left || episodes_left[k] > 0) && (uint32_t)actions[t * B + k] >= n)
          return fail(BSB_INVALID_ARGUMENT, "action " + std::to_string(actions[t * B + k]) + " of active lane " +
                                                std::to_string(k) + (rollout ? " at step " + std::to_string(t) : "") +
                                                " is outside [0, " + std::to_string(n) + ")");
  }
  LaunchArgs a = make_args(env, out, mode == MODE_STEP ? actions : nullptr, T, mode);
  a.action_seed = action_seed; a.actions_out = actions_out;
  int rc = run(env, a, static_cast<cudaStream_t>(stream), nullptr, mask, episodes_left, mask_out, previous, policy,
               replay, sequence, ensemble);
  if (rc == BSB_OK) advance_steps(env, T);
  return rc;
}

int32_t bsb_reset_masked(bsb_env* env, const uint8_t* mask, const bsb_outputs* out, void* stream) {
  if (!env || !mask || !out || !out->observation)
    return fail(BSB_INVALID_ARGUMENT, "bsb_reset_masked needs a mask and outputs with an observation buffer");
  return masked_call(env, nullptr, mask, out, stream, MODE_RESET);
}

int32_t bsb_step_masked(bsb_env* env, const int32_t* actions, const uint8_t* mask, const bsb_outputs* out, void* stream) {
  if (!env || !actions || !mask || !out || !out->observation)
    return fail(BSB_INVALID_ARGUMENT, "bsb_step_masked needs actions, a mask and outputs with an observation buffer");
  return masked_call(env, actions, mask, out, stream, MODE_STEP);
}

int32_t bsb_rollout(bsb_env* env, int64_t num_steps, const int32_t* actions, uint64_t action_seed,
                    const bsb_outputs* out, int32_t* actions_out, void* stream) {
  if (!env || !out || !out->observation) return fail(BSB_INVALID_ARGUMENT, "bsb_rollout needs outputs with an observation buffer");
  if (num_steps <= 0) return fail(BSB_INVALID_ARGUMENT, "num_steps must be positive");
  { int crc = check_final_observation(env, out); if (crc != BSB_OK) return crc; }
  { int frc = drain_host_steps(env); if (frc != BSB_OK) return frc; }
  if (env->device < 0 && actions) { int vrc = check_host_actions(env, actions, num_steps * env->p.batch); if (vrc != BSB_OK) return vrc; }
  LaunchArgs a = make_args(env, out, actions, num_steps, MODE_STEP);
  a.action_seed = action_seed; a.actions_out = actions_out;
  int rc = run(env, a, static_cast<cudaStream_t>(stream));
  if (rc == BSB_OK) advance_steps(env, num_steps);
  return rc;
}

int32_t bsb_rollout_masked(bsb_env* env, int64_t num_steps, const int32_t* actions, uint64_t action_seed,
                           const uint8_t* mask, int64_t* episodes_left, const bsb_outputs* out, int32_t* actions_out,
                           void* stream) {
  if (!env || !mask || !out || !out->observation)
    return fail(BSB_INVALID_ARGUMENT, "bsb_rollout_masked needs a mask and outputs with an observation buffer");
  if (num_steps <= 0) return fail(BSB_INVALID_ARGUMENT, "num_steps must be positive");
  return masked_call(env, actions, mask, out, stream, MODE_STEP, num_steps, true, action_seed, actions_out, episodes_left);
}

// bsb_rollout_masked of sampled actions with no outputs: a launch without an observation buffer takes masked_kernel's
// CALL_ADVANCE instantiation (run_masked), and the host path renders nothing.
int32_t bsb_advance_masked(bsb_env* env, int64_t num_steps, uint64_t action_seed, const uint8_t* mask,
                           int64_t* episodes_left, void* stream) {
  if (!env || !mask) return fail(BSB_INVALID_ARGUMENT, "bsb_advance_masked needs a handle and a mask");
  if (num_steps <= 0) return fail(BSB_INVALID_ARGUMENT, "num_steps must be positive");
  bsb_outputs none;
  memset(&none, 0, sizeof(none));
  return masked_call(env, nullptr, mask, &none, stream, MODE_STEP, num_steps, true, action_seed, nullptr, episodes_left);
}

// One masked step with budgets that first keeps the masked-in lanes' current outputs in `previous`: masked_kernel's
// CALL_BUDGETED instantiation (run_masked), or host_budgeted on a host handle.  The mask is cleared in place one call
// after a lane's budget is spent.
// The refusals bsb_step_budgeted, bsb_step_budgeted_policy, bsb_step_budgeted_record and bsb_step_budgeted_sequence
// share (`choice`: the actions or the policy).
static int check_budgeted(const bsb_env* env, const void* choice, const uint8_t* mask, const int64_t* episodes_left,
                          const bsb_outputs* out, const bsb_outputs* previous, const std::string& name,
                          const char* what) {
  if (!env || !choice || !mask || !episodes_left || !out || !previous || !out->observation || !previous->observation)
    return fail(BSB_INVALID_ARGUMENT, name + " needs " + what + ", a mask, budgets and two output sets with "
                                      "observation buffers");
  if (previous->observation == out->observation)
    return fail(BSB_INVALID_ARGUMENT, name + " needs `previous` to have its own observation buffer");
  if (!out->final_observation != !previous->final_observation)
    return fail(BSB_INVALID_ARGUMENT, "final_observation must be set in both output sets or in neither");
  return check_final_observation(env, previous);
}

// The refusals of a policy (bsb_step_budgeted_policy, bsb_step_budgeted_record, bsb_step_budgeted_sequence).
static int check_policy(const bsb_policy* policy, const std::string& name) {
  if (!policy->values) return fail(BSB_INVALID_ARGUMENT, name + " needs the policy's values");
  if (policy->kind != BSB_POLICY_EPSILON_GREEDY && policy->kind != BSB_POLICY_SOFTMAX)
    return fail(BSB_INVALID_ARGUMENT, "unknown policy kind " + std::to_string(policy->kind));
  if (policy->reserved != 0) return fail(BSB_INVALID_ARGUMENT, "bsb_policy.reserved must be 0");
  if (policy->kind == BSB_POLICY_EPSILON_GREEDY && !(policy->epsilon >= 0.0 && policy->epsilon <= 1.0))
    return fail(BSB_INVALID_ARGUMENT, "epsilon must lie in [0, 1], got " + std::to_string(policy->epsilon));
  if (policy->kind == BSB_POLICY_SOFTMAX && policy->epsilon != 0.0)
    return fail(BSB_INVALID_ARGUMENT, "a softmax policy takes no epsilon: it must be 0");
  return BSB_OK;
}

int32_t bsb_step_budgeted(bsb_env* env, const int32_t* actions, uint8_t* mask, int64_t* episodes_left,
                          const bsb_outputs* out, const bsb_outputs* previous, void* stream) {
  { int rc = check_budgeted(env, actions, mask, episodes_left, out, previous, "bsb_step_budgeted", "actions"); if (rc != BSB_OK) return rc; }
  return masked_call(env, actions, mask, out, stream, MODE_STEP, 1, false, 0, nullptr, episodes_left, mask, previous);
}

// bsb_step_budgeted with each stepping lane's action chosen from its row of policy->values on the policy stream:
// masked_kernel's CALL_POLICY instantiation (run_masked), or host_policy on a host handle.
int32_t bsb_step_budgeted_policy(bsb_env* env, const bsb_policy* policy, uint8_t* mask, int64_t* episodes_left,
                                 const bsb_outputs* out, const bsb_outputs* previous, int32_t* actions_out,
                                 void* stream) {
  const std::string name = "bsb_step_budgeted_policy";
  { int rc = check_budgeted(env, policy, mask, episodes_left, out, previous, name, "a policy"); if (rc != BSB_OK) return rc; }
  { int rc = check_policy(policy, name); if (rc != BSB_OK) return rc; }
  return masked_call(env, nullptr, mask, out, stream, MODE_STEP, 1, false, 0, actions_out, episodes_left, mask, previous,
                     policy);
}

// The refusals a replay ring (`batch`: a sample's output, which has no counts) shares between the recorded step and
// the sampler.
static int check_ring(const bsb_replay* r, const std::string& name, const char* what, bool batch) {
  if (!r || !r->obs_tm1 || !r->action || !r->next.observation || (!batch && !r->num_added))
    return fail(BSB_INVALID_ARGUMENT, name + " needs " + what + " with obs_tm1, action, next.observation" +
                                          (batch ? "" : " and num_added"));
  if (batch && r->num_added) return fail(BSB_INVALID_ARGUMENT, name + ": a sample's batch has no num_added (NULL)");
  if (r->capacity < 1 || r->capacity > INT32_MAX)
    return fail(BSB_INVALID_ARGUMENT, name + ": capacity must lie in [1, 2^31 - 1], got " + std::to_string(r->capacity));
  if (r->next.final_observation)
    return fail(BSB_INVALID_ARGUMENT, name + ": a ring keeps no final observations (next.final_observation must be NULL)");
  if (r->obs_tm1 == r->next.observation)
    return fail(BSB_INVALID_ARGUMENT, name + ": obs_tm1 and next.observation must be separate buffers");
  return BSB_OK;
}

// The refusals of a replay a step appends to (bsb_step_budgeted_record, bsb_step_budgeted_ensemble).
static int check_record(const bsb_env* env, const bsb_outputs* out, const bsb_outputs* previous, const bsb_replay* replay,
                        const std::string& name) {
  { int rc = check_ring(replay, name, "a replay", false); if (rc != BSB_OK) return rc; }
  if (!out->step_type || !out->discount || (!out->reward && !out->reward_f64))
    return fail(BSB_INVALID_ARGUMENT, name + " needs out's step_type, discount and reward (or reward_f64)");
  for (const float* ring : {replay->obs_tm1, replay->next.observation})
    if (ring == out->observation || ring == previous->observation || (out->final_observation && ring == out->final_observation))
      return fail(BSB_INVALID_ARGUMENT, name + ": a ring observation buffer must not be out's or previous's");
  if (env->same_step && !out->final_observation)
    return fail(BSB_INVALID_ARGUMENT, name + " on a same-step handle needs out->final_observation: it is o_t of a LAST");
  return BSB_OK;
}

// bsb_step_budgeted or bsb_step_budgeted_policy that appends each transition to its lane's ring: masked_kernel's
// CALL_RECORD instantiation (run_masked), or host_record on a host handle.
int32_t bsb_step_budgeted_record(bsb_env* env, const int32_t* actions, const bsb_policy* policy, uint8_t* mask,
                                 int64_t* episodes_left, const bsb_outputs* out, const bsb_outputs* previous,
                                 int32_t* actions_out, const bsb_replay* replay, void* stream) {
  const std::string name = "bsb_step_budgeted_record";
  if (!actions == !policy) return fail(BSB_INVALID_ARGUMENT, name + " takes actions or a policy: exactly one of them");
  const void* choice = actions ? static_cast<const void*>(actions) : static_cast<const void*>(policy);
  { int rc = check_budgeted(env, choice, mask, episodes_left, out, previous, name, actions ? "actions" : "a policy"); if (rc != BSB_OK) return rc; }
  if (policy) { int rc = check_policy(policy, name); if (rc != BSB_OK) return rc; }
  else if (actions_out) return fail(BSB_INVALID_ARGUMENT, name + ": actions_out reports a policy's picks: pass NULL with actions");
  { int rc = check_record(env, out, previous, replay, name); if (rc != BSB_OK) return rc; }
  return masked_call(env, actions, mask, out, stream, MODE_STEP, 1, false, 0, actions_out, episodes_left, mask, previous,
                     policy, replay);
}

// bsb_step_budgeted or bsb_step_budgeted_policy that appends each transition to its lane's sequence buffer:
// masked_sequence_kernel (CALL_SEQUENCE, run_masked), or host_sequence on a host handle.
int32_t bsb_step_budgeted_sequence(bsb_env* env, const int32_t* actions, const bsb_policy* policy, uint8_t* mask,
                                   int64_t* episodes_left, const bsb_outputs* out, const bsb_outputs* previous,
                                   int32_t* actions_out, const bsb_sequence* sequence, void* stream) {
  const std::string name = "bsb_step_budgeted_sequence";
  if (!actions == !policy) return fail(BSB_INVALID_ARGUMENT, name + " takes actions or a policy: exactly one of them");
  const void* choice = actions ? static_cast<const void*>(actions) : static_cast<const void*>(policy);
  { int rc = check_budgeted(env, choice, mask, episodes_left, out, previous, name, actions ? "actions" : "a policy"); if (rc != BSB_OK) return rc; }
  if (policy) { int rc = check_policy(policy, name); if (rc != BSB_OK) return rc; }
  else if (actions_out) return fail(BSB_INVALID_ARGUMENT, name + ": actions_out reports a policy's picks: pass NULL with actions");
  const bsb_sequence* q = sequence;
  if (!q || !q->length || !q->ready || !q->observations || !q->action || !q->next.step_type || !q->next.discount ||
      (!q->next.reward && !q->next.reward_f64))
    return fail(BSB_INVALID_ARGUMENT, name + " needs a sequence with length, ready, observations, action and next's "
                                             "step_type, discount and reward (or reward_f64)");
  if (q->max_length < 1 || q->max_length > INT32_MAX)
    return fail(BSB_INVALID_ARGUMENT, name + ": max_length must lie in [1, 2^31 - 1], got " + std::to_string(q->max_length));
  if (q->next.observation || q->next.final_observation)
    return fail(BSB_INVALID_ARGUMENT, name + ": a sequence keeps its observations in `observations` (next.observation "
                                             "and next.final_observation must be NULL)");
  if (!out->step_type || !out->discount || (!out->reward && !out->reward_f64))
    return fail(BSB_INVALID_ARGUMENT, name + " needs out's step_type, discount and reward (or reward_f64)");
  if (q->observations == out->observation || q->observations == previous->observation ||
      (out->final_observation && q->observations == out->final_observation))
    return fail(BSB_INVALID_ARGUMENT, name + ": the sequence's observation buffer must not be out's or previous's");
  if (env->same_step && !out->final_observation)
    return fail(BSB_INVALID_ARGUMENT, name + " on a same-step handle needs out->final_observation: it is o_t of a LAST");
  return masked_call(env, actions, mask, out, stream, MODE_STEP, 1, false, 0, actions_out, episodes_left, mask, previous,
                     policy, nullptr, sequence);
}

// bsb_step_budgeted_policy (no replay) or bsb_step_budgeted_record (a replay) with epsilon-greedy over the rows of
// each lane's active head, which is redrawn when the lane's episode ends: masked_ensemble_kernel (CALL_ENSEMBLE,
// run_masked), or host_ensemble on a host handle.
int32_t bsb_step_budgeted_ensemble(bsb_env* env, const bsb_ensemble_policy* policy, uint8_t* mask,
                                   int64_t* episodes_left, const bsb_outputs* out, const bsb_outputs* previous,
                                   int32_t* actions_out, const bsb_replay* replay, void* stream) {
  const std::string name = "bsb_step_budgeted_ensemble";
  { int rc = check_budgeted(env, policy, mask, episodes_left, out, previous, name, "a policy"); if (rc != BSB_OK) return rc; }
  if (!policy->values || !policy->heads) return fail(BSB_INVALID_ARGUMENT, name + " needs the policy's values and heads");
  if (policy->num_heads < 1 || policy->num_heads > 65536)
    return fail(BSB_INVALID_ARGUMENT, name + ": num_heads must lie in [1, 65536], got " + std::to_string(policy->num_heads));
  if (policy->reserved != 0) return fail(BSB_INVALID_ARGUMENT, "bsb_ensemble_policy.reserved must be 0");
  if (!(policy->epsilon >= 0.0 && policy->epsilon <= 1.0))
    return fail(BSB_INVALID_ARGUMENT, "epsilon must lie in [0, 1], got " + std::to_string(policy->epsilon));
  if (replay) { int rc = check_record(env, out, previous, replay, name); if (rc != BSB_OK) return rc; }
  bsb_policy rule;                       // the rule; its values are the rows of the active heads
  memset(&rule, 0, sizeof(rule));
  rule.kind = BSB_POLICY_EPSILON_GREEDY;
  rule.values = policy->values;
  rule.epsilon = policy->epsilon;
  rule.seed = policy->seed;
  return masked_call(env, nullptr, mask, out, stream, MODE_STEP, 1, false, 0, actions_out, episodes_left, mask, previous,
                     &rule, replay, nullptr, policy);
}

// ----- replay sampling --------------------------------------------------------------------------------------------
namespace bsb {
namespace {

// What one sample gathers (bsb_replay_sample).  Observation rows move as raw bytes: lane i's row is elements
// [row_of(i), row_of(i) + K_i) of every slot of step_elems elements (a ragged pack: its setting's offset and length).
struct SampleArgs {
  const int64_t* num_added;
  const uint8_t* obs_tm1; const uint8_t* obs;
  const int32_t* action; const float* reward; const double* reward_f64; const float* discount; const int32_t* step_type;
  uint8_t* out_tm1; uint8_t* out_obs;
  int32_t* out_action; float* out_reward; double* out_reward_f64; float* out_discount; int32_t* out_step_type;
  uint8_t* ready;
  const RaggedTable* ragged;          // a ragged pack's settings (in the handle's memory space), else null
  int64_t batch, lanes_per_setting, capacity, size, min_size, obs_numel, step_elems;
  int32_t elem_bytes, vec_ok;         // vec_ok: the four observation buffers and every slot start 16-byte aligned
  uint64_t seed, draw, lane_offset;
  int64_t step0;                      // the call index; graph-safe mode adds the device clock
  const unsigned long long* clock;
};

// (filled slots, ready) of lane i, and the first element and length of its observation row within a slot.
BSB_HD void sample_lane(const SampleArgs& s, int64_t i, int64_t& n, bool& ok, int64_t& row, int64_t& K) {
  n = s.num_added[i] < s.capacity ? s.num_added[i] : s.capacity;
  ok = n >= (s.min_size > 1 ? s.min_size : 1);
  row = i * s.obs_numel;
  K = s.obs_numel;
  if (s.ragged) {
    const RaggedSetting& r = ragged_setting(s.ragged, i / s.ragged->pack.lanes_per_setting);
    row = r.obs_offset + (i - r.lane_shift) * (int64_t)r.obs_numel;
    K = r.obs_numel;
  }
}

// The Philox block of samples 4 q .. 4 q + 3 of lane i at call index c: word j & 3 is sample j's.
BSB_HD PhiloxBlock sample_block(const SampleArgs& s, int64_t c, int64_t i, int64_t q) {
  return philox4x64_10((u64)c, s.draw, (u64)q, STREAM_REPLAY, s.seed, s.lane_offset + (u64)(i % s.lanes_per_setting));
}

// Sample j of lane i: slot `slot` of the ring to entry j of the batch.  `tid`, `threads`: this thread's share of the
// row copy (the kernel's warp, or the whole row on the host).
BSB_HD void sample_copy(const SampleArgs& s, int64_t i, int64_t j, int64_t slot, int64_t row, int64_t K, int tid,
                        int threads) {
  const int64_t from = slot * s.batch + i, to = j * s.batch + i;
  if (tid == 0) {
    s.out_action[to] = s.action[from];
    if (s.out_reward) s.out_reward[to] = s.reward[from];
    if (s.out_reward_f64) s.out_reward_f64[to] = s.reward_f64[from];
    if (s.out_discount) s.out_discount[to] = s.discount[from];
    if (s.out_step_type) s.out_step_type[to] = s.step_type[from];
  }
  const int64_t bytes = K * s.elem_bytes;
  const int64_t src = (slot * s.step_elems + row) * s.elem_bytes, dst = (j * s.step_elems + row) * s.elem_bytes;
  if (s.vec_ok && (row * s.elem_bytes) % 16 == 0 && bytes % 16 == 0) {
    for (int64_t q = tid; q < bytes / 16; q += threads) {
      reinterpret_cast<uint4*>(s.out_tm1 + dst)[q] = reinterpret_cast<const uint4*>(s.obs_tm1 + src)[q];
      reinterpret_cast<uint4*>(s.out_obs + dst)[q] = reinterpret_cast<const uint4*>(s.obs + src)[q];
    }
  } else {
    for (int64_t q = tid; q < bytes; q += threads) {
      s.out_tm1[dst + q] = s.obs_tm1[src + q];
      s.out_obs[dst + q] = s.obs[src + q];
    }
  }
}

// One warp per (group of four samples, lane i), lanes fastest: one Philox block for the group's four slots, then per
// sample lane 0 moves the scalars and the warp both rows, with 16-byte loads and stores where the row and the buffers
// allow.
__global__ void __launch_bounds__(256) replay_sample_kernel(const SampleArgs s) {
  const int tid = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int64_t groups = (s.size + 3) / 4, items = groups * s.batch;
  int64_t c = s.step0;
  if (s.clock) c += (int64_t)*reinterpret_cast<const volatile unsigned long long*>(s.clock + 16 * (blockIdx.x % CLOCK_GROUPS));
  for (int64_t item = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); item < items; item += warps) {
    const int64_t q = item / s.batch, i = item - q * s.batch;
    int64_t n, row, K;
    bool ok;
    sample_lane(s, i, n, ok, row, K);
    if (q == 0 && tid == 0 && s.ready) s.ready[i] = ok ? 1 : 0;
    if (!ok) continue;
    const PhiloxBlock b = sample_block(s, c, i, q);
    for (int64_t j = 4 * q; j < 4 * q + 4 && j < s.size; ++j)
      sample_copy(s, i, j, replay_slot(replay_word(b, j), n), row, K, tid, 32);
  }
}

// What a bootstrap sample adds (bsb_replay_sample_bootstrap): SampleArgs grown at its end, passed to
// bootstrap_sample_kernel only, so that replay_sample_kernel compiles as it did.  boot_mask / boot_noise: [size, B, K],
// nullable.
struct BootstrapArgs : SampleArgs {
  uint8_t* boot_mask;
  float* boot_noise;
  double mask_prob;
  uint64_t boot_seed;
  int32_t num_heads;
};

// The bootstrap draws of sample j of lane i (global lane g), which drew ring slot `slot`: the slot's transition index
// t (the lane's (t + 1)-th transition; the ring holds its last min(N, capacity) of N), then every head's mask and
// noise.  `tid`, `threads`: this thread's share of the heads (the kernel's warp, or all of them on the host); a mask
// thread draws one Philox block for four heads, a noise thread one head.
BSB_HD void bootstrap_draws(const BootstrapArgs& s, int64_t i, int64_t j, int64_t slot, u64 g, int tid, int threads) {
  const int64_t N = s.num_added[i];
  const int64_t t = N - 1 - (N - 1 - slot) % s.capacity;
  const int64_t base = (j * s.batch + i) * (int64_t)s.num_heads;
  if (s.boot_mask) {
    const bool draw = s.mask_prob > 0.0 && s.mask_prob < 1.0;      // else every draw gives mask_prob itself
    for (int64_t q = tid; 4 * q < s.num_heads; q += threads) {
      PhiloxBlock b = {0, 0, 0, 0};
      if (draw) b = bootstrap_mask_block(s.boot_seed, g, (u64)t, (u64)q);
      for (int64_t k = 4 * q; k < 4 * q + 4 && k < s.num_heads; ++k)
        s.boot_mask[base + k] = draw ? bootstrap_mask_word(replay_word(b, k), s.mask_prob) : (s.mask_prob >= 1.0 ? 1 : 0);
    }
  }
  if (s.boot_noise)
    for (int64_t k = tid; k < s.num_heads; k += threads) s.boot_noise[base + k] = bootstrap_noise(s.boot_seed, g, (u64)t, (u64)k);
}

// replay_sample_kernel with the bootstrap draws of every sample it gathers: one warp per (group of four samples, lane
// i), the heads' draws spread over the warp's threads.
__global__ void __launch_bounds__(256) bootstrap_sample_kernel(const BootstrapArgs s) {
  const int tid = threadIdx.x & 31;
  const int64_t warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  const int64_t groups = (s.size + 3) / 4, items = groups * s.batch;
  int64_t c = s.step0;
  if (s.clock) c += (int64_t)*reinterpret_cast<const volatile unsigned long long*>(s.clock + 16 * (blockIdx.x % CLOCK_GROUPS));
  for (int64_t item = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); item < items; item += warps) {
    const int64_t q = item / s.batch, i = item - q * s.batch;
    int64_t n, row, K;
    bool ok;
    sample_lane(s, i, n, ok, row, K);
    if (q == 0 && tid == 0 && s.ready) s.ready[i] = ok ? 1 : 0;
    if (!ok) continue;
    const PhiloxBlock b = sample_block(s, c, i, q);
    const u64 g = s.lane_offset + (u64)(i % s.lanes_per_setting);
    for (int64_t j = 4 * q; j < 4 * q + 4 && j < s.size; ++j) {
      const int64_t slot = replay_slot(replay_word(b, j), n);
      sample_copy(s, i, j, slot, row, K, tid, 32);
      bootstrap_draws(s, i, j, slot, g, tid, 32);
    }
  }
}

// bsb_replay_sample on a host handle: the kernel's gather, lane by lane; with `boot`
// (bsb_replay_sample_bootstrap), bootstrap_sample_kernel's draws too.
void host_sample(const SampleArgs& s, const BootstrapArgs* boot = nullptr) {
  for (int64_t i = 0; i < s.batch; ++i) {
    int64_t n, row, K;
    bool ok;
    sample_lane(s, i, n, ok, row, K);
    if (s.ready) s.ready[i] = ok ? 1 : 0;
    if (!ok) continue;
    for (int64_t q = 0; 4 * q < s.size; ++q) {
      const PhiloxBlock b = sample_block(s, s.step0, i, q);
      for (int64_t j = 4 * q; j < 4 * q + 4 && j < s.size; ++j) {
        const int64_t slot = replay_slot(replay_word(b, j), n);
        sample_copy(s, i, j, slot, row, K, 0, 1);
        if (boot) bootstrap_draws(*boot, i, j, slot, s.lane_offset + (u64)(i % s.lanes_per_setting), 0, 1);
      }
    }
  }
}

}  // namespace
}  // namespace bsb

// bsb_replay_sample (`bootstrap` null: replay_sample_kernel) and bsb_replay_sample_bootstrap
// (bootstrap_sample_kernel), or host_sample on a host handle.
static int sample_call(bsb_env* env, const bsb_replay* replay, int64_t size, int64_t min_size, uint64_t seed,
                       uint64_t draw, const bsb_replay* batch, uint8_t* ready, const bsb_bootstrap* bootstrap,
                       void* stream, const std::string& name) {
  if (!env) return fail(BSB_INVALID_ARGUMENT, name + " needs a handle");
  if (size <= 0) return fail(BSB_INVALID_ARGUMENT, name + ": size must be positive, got " + std::to_string(size));
  if (min_size < 0) return fail(BSB_INVALID_ARGUMENT, name + ": min_size must not be negative, got " + std::to_string(min_size));
  { int rc = check_ring(replay, name, "a replay", false); if (rc != BSB_OK) return rc; }
  { int rc = check_ring(batch, name, "a batch", true); if (rc != BSB_OK) return rc; }
  if (batch->capacity != size)
    return fail(BSB_INVALID_ARGUMENT, name + ": the batch's capacity must equal size (" + std::to_string(size) + "), got " +
                                          std::to_string(batch->capacity));
  if ((batch->next.reward && !replay->next.reward) || (batch->next.reward_f64 && !replay->next.reward_f64) ||
      (batch->next.discount && !replay->next.discount) || (batch->next.step_type && !replay->next.step_type))
    return fail(BSB_INVALID_ARGUMENT, name + ": the batch asks for a scalar the ring does not carry");
  if (bootstrap) {
    if (bootstrap->num_heads < 1 || bootstrap->num_heads > 65536)
      return fail(BSB_INVALID_ARGUMENT, name + ": num_heads must lie in [1, 65536], got " + std::to_string(bootstrap->num_heads));
    if (bootstrap->reserved != 0) return fail(BSB_INVALID_ARGUMENT, "bsb_bootstrap.reserved must be 0");
    if (!(bootstrap->mask_prob >= 0.0 && bootstrap->mask_prob <= 1.0))
      return fail(BSB_INVALID_ARGUMENT, name + ": mask_prob must lie in [0, 1], got " + std::to_string(bootstrap->mask_prob));
    if (!bootstrap->mask && !bootstrap->noise)
      return fail(BSB_INVALID_ARGUMENT, name + " needs the bootstrap's mask or noise buffer (or both)");
  }
  { int frc = drain_host_steps(env); if (frc != BSB_OK) return frc; }
  BootstrapArgs boot;                    // s, grown by the bootstrap draws
  memset(&boot, 0, sizeof(boot));
  SampleArgs& s = boot;
  s.num_added = replay->num_added;
  s.obs_tm1 = reinterpret_cast<const uint8_t*>(replay->obs_tm1);
  s.obs = reinterpret_cast<const uint8_t*>(replay->next.observation);
  s.action = replay->action; s.reward = replay->next.reward; s.reward_f64 = replay->next.reward_f64;
  s.discount = replay->next.discount; s.step_type = replay->next.step_type;
  s.out_tm1 = reinterpret_cast<uint8_t*>(batch->obs_tm1);
  s.out_obs = reinterpret_cast<uint8_t*>(batch->next.observation);
  s.out_action = batch->action; s.out_reward = batch->next.reward; s.out_reward_f64 = batch->next.reward_f64;
  s.out_discount = batch->next.discount; s.out_step_type = batch->next.step_type;
  s.ready = ready;
  s.ragged = env->ragged ? reinterpret_cast<const RaggedTable*>(env->p.pack) : nullptr;
  s.batch = env->p.batch; s.lanes_per_setting = env->lanes_per_setting;
  s.capacity = replay->capacity; s.size = size; s.min_size = min_size;
  s.obs_numel = env->p.obs_numel; s.step_elems = env->step_elems; s.elem_bytes = env->obs_elem_bytes;
  s.vec_ok = ((size_t)env->step_elems * (size_t)env->obs_elem_bytes) % 16 == 0;
  for (const float* buf : {replay->obs_tm1, replay->next.observation, batch->obs_tm1, batch->next.observation})
    if (reinterpret_cast<uintptr_t>(buf) % 16 != 0) s.vec_ok = 0;
  s.seed = seed; s.draw = draw; s.lane_offset = env->p.lane_offset;
  s.step0 = env->steps_done;
  if (bootstrap) {
    boot.boot_mask = bootstrap->mask;
    boot.boot_noise = bootstrap->noise;
    boot.mask_prob = bootstrap->mask_prob;
    boot.boot_seed = bootstrap->seed;
    boot.num_heads = bootstrap->num_heads;
  }
  if (env->device < 0) { host_sample(s, bootstrap ? &boot : nullptr); return BSB_OK; }
  DeviceGuard guard(env->device);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaStreamCaptureStatus capture = cudaStreamCaptureStatusNone;
  BSB_CUDA(cudaStreamIsCapturing(st, &capture));
  if (capture != cudaStreamCaptureStatusNone) env->graph_safe = true;
  if (env->graph_safe) s.clock = env->clock;
  const int64_t warps = (size + 3) / 4 * s.batch;
  int64_t grid = (warps + 7) / 8;
  const int64_t cap = (int64_t)env->num_sms * 64;
  if (grid > cap) grid = cap;
  if (bootstrap) bootstrap_sample_kernel<<<(unsigned)grid, 256, 0, st>>>(boot);
  else replay_sample_kernel<<<(unsigned)grid, 256, 0, st>>>(s);
  BSB_CUDA(cudaGetLastError());
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return BSB_OK;
}

int32_t bsb_replay_sample(bsb_env* env, const bsb_replay* replay, int64_t size, int64_t min_size, uint64_t seed,
                          uint64_t draw, const bsb_replay* batch, uint8_t* ready, void* stream) {
  return sample_call(env, replay, size, min_size, seed, draw, batch, ready, nullptr, stream, "bsb_replay_sample");
}

int32_t bsb_replay_sample_bootstrap(bsb_env* env, const bsb_replay* replay, int64_t size, int64_t min_size,
                                    uint64_t seed, uint64_t draw, const bsb_replay* batch, uint8_t* ready,
                                    const bsb_bootstrap* bootstrap, void* stream) {
  const std::string name = "bsb_replay_sample_bootstrap";
  if (!bootstrap) return fail(BSB_INVALID_ARGUMENT, name + " needs a bootstrap");
  return sample_call(env, replay, size, min_size, seed, draw, batch, ready, bootstrap, stream, name);
}

int32_t bsb_random_actions(uint64_t action_seed, uint64_t lane_offset, int64_t batch, int64_t first_step,
                           int64_t num_steps, int32_t num_actions, int32_t* out) {
  if (!out || batch <= 0 || num_steps <= 0 || num_actions <= 0) return fail(BSB_INVALID_ARGUMENT, "bad arguments");
  for (int64_t t = 0; t < num_steps; ++t)
    for (int64_t i = 0; i < batch; ++i)
      out[t * batch + i] = sample_action(action_seed, lane_offset + (uint64_t)i, (uint64_t)(first_step + t), num_actions);
  return BSB_OK;
}

int32_t bsb_info_count(const bsb_env* env, int32_t* count) {
  if (!env || !count) return fail(BSB_INVALID_ARGUMENT, "null argument");
  *count = env->names.n; return BSB_OK;
}
const char* bsb_info_name(const bsb_env* env, int32_t index) {
  if (!env || index < 0 || index >= env->names.n) return nullptr;
  return env->names.names[index];
}

static int copy_field(bsb_env* env, const double* src, double* dst, void* stream) {
  const size_t bytes = (size_t)env->p.batch * sizeof(double);
  if (env->device >= 0) {
    DeviceGuard guard(env->device);
    BSB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
  } else {
    memcpy(dst, src, bytes);
  }
  return BSB_OK;
}

int32_t bsb_read_info(bsb_env* env, int32_t index, double* dst, void* stream) {
  if (!env || !dst) return fail(BSB_INVALID_ARGUMENT, "null argument");
  if (index < 0 || index >= env->names.n) return fail(BSB_INVALID_ARGUMENT, "info index out of range");
  { int frc = drain_host_steps(env); if (frc != BSB_OK) return frc; }
  return copy_field(env, env->p.info + (size_t)index * (size_t)env->p.batch, dst, stream);
}

int32_t bsb_read_episode_stats(bsb_env* env, int32_t field, double* dst, void* stream) {
  if (!env || !dst) return fail(BSB_INVALID_ARGUMENT, "null argument");
  if (!env->p.ep) return fail(BSB_INVALID_ARGUMENT, "environment was created without BSB_FLAG_TRACK_EPISODES");
  if (field < 0 || field >= 5) return fail(BSB_INVALID_ARGUMENT, "episode-stat field out of range");
  { int frc = drain_host_steps(env); if (frc != BSB_OK) return frc; }
  const int64_t B = env->p.batch;
  if (env->device >= 0) {
    DeviceGuard guard(env->device);
    episode_stat_kernel<<<(unsigned)((B + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(env->p, field, env->steps_done, env->graph_safe ? env->clock : nullptr, dst);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    BSB_CUDA(cudaGetLastError());
  } else {
    for (int64_t i = 0; i < B; ++i) dst[i] = episode_stat(env->p, i, field, env->steps_done);
  }
  return BSB_OK;
}

// The rows of `env`: one for the whole handle, or one per setting (an ordinary handle has one setting).
static int32_t sum_rows(const bsb_env* env, bool per_setting) { return per_setting ? env->n_settings : 1; }

// Fills the job of `env` (whole handle or per setting) at jobs.job[k], its first row at `row`.
static void put_sum_job(SumJobs& jobs, int32_t k, int32_t row, const bsb_env* env, bool per_setting) {
  SumJob& j = jobs.job[k];
  j.ep = env->p.ep; j.batch = env->p.batch; j.calls = env->steps_done;
  j.lanes = per_setting ? env->lanes_per_setting : env->p.batch;
  j.n_settings = sum_rows(env, per_setting);
  j.clock = env->graph_safe ? env->clock : nullptr; j.scratch = env->sum_scratch;
  jobs.row_start[k] = row;
}

// The host path: each row's lanes in order from 0.0.
static void host_sums(const bsb_env* env, bool per_setting, double* dst) {
  const int64_t lanes = per_setting ? env->lanes_per_setting : env->p.batch;
  for (int32_t r = 0; r < sum_rows(env, per_setting); ++r)
    for (int f = 0; f < 5; ++f) {
      double s = 0.0;
      for (int64_t i = r * lanes; i < (r + 1) * lanes; ++i) s += episode_stat(env->p, i, f, env->steps_done);
      dst[5 * r + f] = s;
    }
}

// Shared validation of the list calls: null handles, untracked handles, mixed devices, a repeated handle.
static int32_t check_sum_list(bsb_env* const* envs, int32_t count, const double* dst) {
  if (!envs || !dst || count <= 0) return fail(BSB_INVALID_ARGUMENT, "bad arguments");
  for (int32_t k = 0; k < count; ++k) {
    if (!envs[k]) return fail(BSB_INVALID_ARGUMENT, "null environment");
    if (!envs[k]->p.ep) return fail(BSB_INVALID_ARGUMENT, "environment was created without BSB_FLAG_TRACK_EPISODES");
    if (envs[k]->device != envs[0]->device) return fail(BSB_INVALID_ARGUMENT, "environments live on different devices");
  }
  // Two grid rows of one handle would share its partials and its ticket: the last-block test could then fire before
  // every block of either row has written.  Refused on both paths, so they answer alike.
  std::vector<bsb_env*> seen(envs, envs + count);
  std::sort(seen.begin(), seen.end());
  if (std::adjacent_find(seen.begin(), seen.end()) != seen.end())
    return fail(BSB_INVALID_ARGUMENT, "the same environment is given twice");
  return BSB_OK;
}

// The rows of up to kSumManyMax validated handles of one device in ONE launch of `blocks` x rows blocks.
static int32_t launch_sums(bsb_env* const* envs, int32_t count, bool per_setting, int64_t blocks, double* dst,
                           void* stream) {
  SumJobs jobs;
  memset(&jobs, 0, sizeof(jobs));
  int32_t rows = 0;
  for (int32_t k = 0; k < count; ++k) {
    { int frc = drain_host_steps(envs[k]); if (frc != BSB_OK) return frc; }
    put_sum_job(jobs, k, rows, envs[k], per_setting);
    rows += sum_rows(envs[k], per_setting);
  }
  jobs.count = count;
  DeviceGuard guard(envs[0]->device);
  episode_sum_many_kernel<<<dim3((unsigned)blocks, (unsigned)rows), kSumThreads, 0, static_cast<cudaStream_t>(stream)>>>(jobs, dst);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  BSB_CUDA(cudaGetLastError());
  return BSB_OK;
}

int32_t bsb_sum_episode_stats(bsb_env* env, double* dst5, void* stream) {
  if (!env || !dst5) return fail(BSB_INVALID_ARGUMENT, "null argument");
  if (!env->p.ep) return fail(BSB_INVALID_ARGUMENT, "environment was created without BSB_FLAG_TRACK_EPISODES");
  if (env->device >= 0) {
    int64_t blocks = (env->p.batch + kSumThreads - 1) / kSumThreads;
    if (blocks > kSumBlocks) blocks = kSumBlocks;
    return launch_sums(&env, 1, false, blocks, dst5, stream);
  }
  { int frc = drain_host_steps(env); if (frc != BSB_OK) return frc; }
  host_sums(env, false, dst5);
  return BSB_OK;
}

// bsb_sum_episode_stats_many (per_setting false) and bsb_sum_setting_stats (true).
static int32_t sum_list(bsb_env* const* envs, int32_t count, bool per_setting, double* dst, void* stream) {
  { int rc = check_sum_list(envs, count, dst); if (rc != BSB_OK) return rc; }
  if (envs[0]->device < 0 || count > kSumManyMax) {       // host path / oversized lists: one environment at a time
    for (int32_t k = 0; k < count; ++k) {
      int rc = envs[k]->device < 0 ? drain_host_steps(envs[k])
                                    : launch_sums(envs + k, 1, per_setting, kSumBlocks, dst, stream);
      if (rc != BSB_OK) return rc;
      if (envs[k]->device < 0) host_sums(envs[k], per_setting, dst);
      dst += 5 * sum_rows(envs[k], per_setting);
    }
    return BSB_OK;
  }
  return launch_sums(envs, count, per_setting, kSumBlocks, dst, stream);
}

int32_t bsb_sum_episode_stats_many(bsb_env* const* envs, int32_t count, double* dst, void* stream) {
  return sum_list(envs, count, false, dst, stream);
}

int32_t bsb_sum_setting_stats(bsb_env* const* envs, int32_t count, double* dst, void* stream) {
  return sum_list(envs, count, true, dst, stream);
}

int32_t bsb_log_layout(const bsb_env* env, int32_t* n_points, int32_t* n_columns) {
  if (!env || !n_points || !n_columns) return fail(BSB_INVALID_ARGUMENT, "null argument");
  *n_points = env->p.n_log_points; *n_columns = env->p.log_rows ? 5 + env->names.n : 0;
  return BSB_OK;
}

int32_t bsb_read_log_rows(bsb_env* env, double* rows, int32_t* counts, void* stream) {
  if (!env || !rows || !counts) return fail(BSB_INVALID_ARGUMENT, "null argument");
  if (!env->p.log_rows) return fail(BSB_INVALID_ARGUMENT, "environment was created without a log schedule");
  { int frc = drain_host_steps(env); if (frc != BSB_OK) return frc; }
  const size_t B = (size_t)env->p.batch;
  const size_t row_bytes = (size_t)env->p.n_log_points * (size_t)(5 + env->names.n) * B * sizeof(double);
  if (env->device >= 0) {
    DeviceGuard guard(env->device);
    BSB_CUDA(cudaMemcpyAsync(rows, env->p.log_rows, row_bytes, cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
    BSB_CUDA(cudaMemcpyAsync(counts, env->p.log_next, B * sizeof(int32_t), cudaMemcpyDeviceToDevice, static_cast<cudaStream_t>(stream)));
  } else {
    memcpy(rows, env->p.log_rows, row_bytes);
    memcpy(counts, env->p.log_next, B * sizeof(int32_t));
  }
  return BSB_OK;
}

int32_t bsb_state_bytes(const bsb_env* env, int64_t* nbytes) {
  if (!env || !nbytes) return fail(BSB_INVALID_ARGUMENT, "null argument");
  size_t total = sizeof(int64_t);
  for (size_t k = 0; k < env->state_blocks.size(); ++k) total += env->state_blocks[k].second;
  *nbytes = (int64_t)total; return BSB_OK;
}

int32_t bsb_get_state(bsb_env* env, void* dst_host, int64_t nbytes, void* stream) {
  int64_t need = 0;
  if (!env || !dst_host) return fail(BSB_INVALID_ARGUMENT, "null argument");
  bsb_state_bytes(env, &need);
  if (nbytes != need) return fail(BSB_INVALID_ARGUMENT, "state buffer has the wrong size");
  { int frc = drain_host_steps(env); if (frc != BSB_OK) return frc; }
  DeviceGuard guard(env->device);
  char* dst = static_cast<char*>(dst_host);
  if (env->device >= 0) BSB_CUDA(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
  int64_t steps = 0;
  { int rc = current_steps(env, &steps); if (rc != BSB_OK) return rc; }
  memcpy(dst, &steps, sizeof(int64_t)); dst += sizeof(int64_t);
  for (size_t k = 0; k < env->state_blocks.size(); ++k) {
    if (env->device >= 0) BSB_CUDA(cudaMemcpy(dst, env->state_blocks[k].first, env->state_blocks[k].second, cudaMemcpyDeviceToHost));
    else memcpy(dst, env->state_blocks[k].first, env->state_blocks[k].second);
    dst += env->state_blocks[k].second;
  }
  return BSB_OK;
}

int32_t bsb_set_state(bsb_env* env, const void* src_host, int64_t nbytes, void* stream) {
  int64_t need = 0;
  if (!env || !src_host) return fail(BSB_INVALID_ARGUMENT, "null argument");
  bsb_state_bytes(env, &need);
  if (nbytes != need) return fail(BSB_INVALID_ARGUMENT, "state buffer has the wrong size");
  { int frc = drain_host_steps(env); if (frc != BSB_OK) return frc; }
  DeviceGuard guard(env->device);
  const char* src = static_cast<const char*>(src_host);
  if (env->device >= 0) BSB_CUDA(cudaStreamSynchronize(static_cast<cudaStream_t>(stream)));
  int64_t restored = 0;
  memcpy(&restored, src, sizeof(int64_t)); src += sizeof(int64_t);
  if (env->graph_safe) {
    // steps_done is baked into the captured launches as their base: it must not move.  The restored count goes
    // into the device clock as an offset from that base (two's complement, so it may be "negative").
    const unsigned long long since = (unsigned long long)restored - (unsigned long long)env->steps_done;
    BSB_CUDA(cudaDeviceSynchronize());
    unsigned long long replicas[CLOCK_GROUPS];
    for (int r = 0; r < CLOCK_GROUPS; ++r) replicas[r] = since;
    BSB_CUDA(cudaMemcpy2D(env->clock, 16 * sizeof(unsigned long long), replicas, sizeof(unsigned long long),
                          sizeof(unsigned long long), CLOCK_GROUPS, cudaMemcpyHostToDevice));
  } else {
    env->steps_done = restored;
  }
  for (size_t k = 0; k < env->state_blocks.size(); ++k) {
    if (env->device >= 0) BSB_CUDA(cudaMemcpy(env->state_blocks[k].first, src, env->state_blocks[k].second, cudaMemcpyHostToDevice));
    else memcpy(env->state_blocks[k].first, src, env->state_blocks[k].second);
    src += env->state_blocks[k].second;
  }
  return BSB_OK;
}

int32_t bsb_invalid_actions(bsb_env* env, int32_t* seen) {
  if (!env || !seen) return fail(BSB_INVALID_ARGUMENT, "null argument");
  *seen = 0;
  if (env->bad_action_host) { *seen = *env->bad_action_host; *env->bad_action_host = 0; }
  return BSB_OK;
}

int32_t bsb_host_timing(bsb_env* env, uint64_t* stamps8) {
  if (!env || !stamps8) return fail(BSB_INVALID_ARGUMENT, "null argument");
  if (!env->mailbox) return fail(BSB_INVALID_ARGUMENT, "no host-driven step has run on this handle");
  for (int k = 0; k < 8; ++k) stamps8[k] = env->mailbox->stamp[k];
  return BSB_OK;
}

int32_t bsb_host_flush(bsb_env* env) {
  if (!env) return fail(BSB_INVALID_ARGUMENT, "null argument");
  return finish_awaited(env);
}

// Reports (and clears) an out-of-range action seen by the kernels of a synchronous host step.
static int report_bad_actions(bsb_env* env) {
  if (env->bad_action_host && *env->bad_action_host) {
    *env->bad_action_host = 0;
    return fail(BSB_INVALID_ARGUMENT, "an action was outside [0, " + std::to_string(env->p.num_actions) +
                                          "): the step was taken with that action clamped into range");
  }
  return BSB_OK;
}

// bsb_step_host (mask null) and bsb_step_host_masked.  A masked step is masked_call's step on the caller's host
// buffers: zero-copy with the mailbox when they are pinned, staged otherwise; with `episodes_left`, a lane whose budget
// is spent after the step has its mask byte cleared (run_masked's `mask_out`, or the loop below on host handles).
static int32_t host_step(bsb_env* env, const int32_t* actions, uint8_t* mask, int64_t* episodes_left,
                         const bsb_outputs* host_out, float* device_obs, void* caller_stream, uint32_t flags) {
  if (!env || !actions || !host_out) return fail(BSB_INVALID_ARGUMENT, "null argument");
  const std::string name = mask ? "bsb_step_host_masked" : "bsb_step_host";
  if (host_out->final_observation) return fail(BSB_UNSUPPORTED, name + " does not deliver final_observation");
  if (env->device < 0) {
    if (!host_out->observation) return fail(BSB_INVALID_ARGUMENT, "a host environment writes observations to host_out->observation");
    if (!mask) return bsb_step(env, actions, host_out, nullptr);
    const int rc = masked_call(env, actions, mask, host_out, nullptr, MODE_STEP, 1, false, 0, nullptr, episodes_left);
    if (rc == BSB_OK && episodes_left)
      for (int64_t k = 0; k < env->p.batch; ++k)
        if (mask[k] && episodes_left[k] <= 0) mask[k] = 0;
    return rc;
  }
  if (!host_out->observation && !device_obs) return fail(BSB_INVALID_ARGUMENT, "need host_out->observation or device_obs");
  if ((flags & BSB_HOST_NO_WAIT) && (flags & BSB_HOST_PRELAUNCH)) return fail(BSB_INVALID_ARGUMENT, "BSB_HOST_NO_WAIT and BSB_HOST_PRELAUNCH exclude each other");
  DeviceGuard guard(env->device);
  { int arc = finish_awaited(env); if (arc != BSB_OK) return arc; }      // one step in flight per handle
  const size_t B = (size_t)env->p.batch;
  const size_t obs_bytes = (size_t)env->step_elems * (size_t)env->obs_elem_bytes;
  if (!env->copy_stream) BSB_CUDA(cudaStreamCreateWithFlags(&env->copy_stream, cudaStreamNonBlocking));
  if (flags & BSB_HOST_ORDER_AFTER_STREAM) {
    // Work the caller enqueued earlier on ITS stream (bsb_reset / bsb_step / bsb_rollout of this handle) must have
    // finished with the lane state before this step touches it: fence the handle's stream behind it.
    { int frc = drain_host_steps(env); if (frc != BSB_OK) return frc; }
    if (!env->order_event) BSB_CUDA(cudaEventCreateWithFlags(&env->order_event, cudaEventDisableTiming));
    BSB_CUDA(cudaEventRecord(env->order_event, static_cast<cudaStream_t>(caller_stream)));
    BSB_CUDA(cudaStreamWaitEvent(env->copy_stream, env->order_event, 0));
  }

  // Zero-copy path: when the caller's action and scalar buffers are PINNED host memory (device-addressable under
  // unified addressing), the transition kernel reads the actions from and writes reward / discount / step_type to
  // host memory directly over PCIe -- 1 MB per step, overlapped with the observation stream -- instead of three
  // separate copies with their launch and DMA latencies before and after the kernel.  A masked step also reads (and
  // writes back) the mask there.
  void* d_actions = mapped_device_pointer(env, actions);
  uint8_t* d_mask = mask ? static_cast<uint8_t*>(mapped_device_pointer(env, mask)) : nullptr;
  void* d_reward = host_out->reward ? mapped_device_pointer(env, host_out->reward) : nullptr;
  void* d_reward64 = host_out->reward_f64 ? mapped_device_pointer(env, host_out->reward_f64) : nullptr;
  void *d_discount = nullptr, *d_step_type = nullptr;
  if (d_reward && scalars_back_to_back(*host_out, B)) {      // one pinned block: one query covers all three
    d_discount = static_cast<float*>(d_reward) + B;
    d_step_type = static_cast<float*>(d_reward) + 2 * B;
  } else {
    d_discount = host_out->discount ? mapped_device_pointer(env, host_out->discount) : nullptr;
    d_step_type = host_out->step_type ? mapped_device_pointer(env, host_out->step_type) : nullptr;
  }
  const bool all_mapped = d_actions && (!mask || d_mask) && (!host_out->reward || d_reward) &&
                          (!host_out->reward_f64 || d_reward64) && (!host_out->discount || d_discount) &&
                          (!host_out->step_type || d_step_type);
  if (all_mapped) {
    if (!device_obs && !env->d_obs) BSB_CUDA(cudaMalloc(&env->d_obs, obs_bytes));
    bsb_outputs dev;
    dev.observation = device_obs ? device_obs : env->d_obs;
    dev.reward = static_cast<float*>(d_reward);
    dev.reward_f64 = static_cast<double*>(d_reward64);
    dev.discount = static_cast<float*>(d_discount);
    dev.step_type = static_cast<int32_t*>(d_step_type);
    dev.final_observation = nullptr;
    const int32_t* dev_actions = static_cast<const int32_t*>(d_actions);
    cudaStream_t zs = env->copy_stream;
    uint8_t* mask_out = episodes_left ? d_mask : nullptr;
    // Completion through the mailbox: the kernel's last CTA stores the ticket into pinned host memory after a
    // system-scope fence and the host spins on that word -- a stream synchronise costs a wake-up per step.
    // Observations copied to the host, graph-safe handles and unaligned observation buffers keep the synchronise.
    const bool spin = !env->graph_safe && !host_out->observation && reinterpret_cast<uintptr_t>(dev.observation) % 16 == 0;
    if (!spin) {
      { int frc = drain_host_steps(env); if (frc != BSB_OK) return frc; }
      int zrc = mask ? masked_call(env, dev_actions, d_mask, &dev, zs, MODE_STEP, 1, false, 0, nullptr, episodes_left, mask_out)
                     : bsb_step(env, dev_actions, &dev, zs);
      if (zrc != BSB_OK) return zrc;
      if (host_out->observation) BSB_CUDA(cudaMemcpyAsync(host_out->observation, dev.observation, obs_bytes, cudaMemcpyDeviceToHost, zs));
      BSB_CUDA(cudaStreamSynchronize(zs));
      return report_bad_actions(env);
    }
    { int mrc = mailbox_open(env); if (mrc != BSB_OK) return mrc; }
    const unsigned long long ticket = ++env->next_ticket;
    if (!mask && family_obs_from_state(env)) {
      // Two-phase step: phase 1 (the transitions of every lane) is all that stands between this launch and the
      // observation stream, and reading 4 B per lane over PCIe from inside the kernel is most of it.  The DMA
      // engine brings the actions over NOW, on a side stream, while the previous step's kernel is still
      // streaming observations; the launch waits for that copy on the device.  (The previous kernel read its
      // actions in phase 1, which ended before its completion word was seen: the buffer is free.)
      if (!env->h2d_actions) BSB_CUDA(cudaMalloc(&env->h2d_actions, B * 4));
      if (!env->h2d_stream) {
        BSB_CUDA(cudaStreamCreateWithFlags(&env->h2d_stream, cudaStreamNonBlocking));
        BSB_CUDA(cudaEventCreateWithFlags(&env->h2d_event, cudaEventDisableTiming));
      }
      BSB_CUDA(cudaMemcpyAsync(env->h2d_actions, actions, B * 4, cudaMemcpyHostToDevice, env->h2d_stream));
      BSB_CUDA(cudaEventRecord(env->h2d_event, env->h2d_stream));
      BSB_CUDA(cudaStreamWaitEvent(zs, env->h2d_event, 0));
      dev_actions = env->h2d_actions;
    }
    { int lrc = mailbox_launch(env, ticket, dev_actions, dev, d_mask, episodes_left, mask_out); if (lrc != BSB_OK) return lrc; }
    if ((flags & BSB_HOST_FENCE_CALLER) && env->early_inflight) {
      // Two-phase step: the observation stores outlive this call.  Fence the caller's stream behind the kernel:
      // whatever the caller enqueues there afterwards sees complete observations.
      if (!env->fence_event) BSB_CUDA(cudaEventCreateWithFlags(&env->fence_event, cudaEventDisableTiming));
      BSB_CUDA(cudaEventRecord(env->fence_event, zs));
      BSB_CUDA(cudaStreamWaitEvent(static_cast<cudaStream_t>(caller_stream), env->fence_event, 0));
    }
    if (flags & BSB_HOST_NO_WAIT) {
      // The completion word is collected by bsb_host_wait (or by whichever entry point of this handle runs next),
      // so the caller can drive ANOTHER handle while this step's scalars cross PCIe.
      env->awaiting_ticket = ticket;
      return BSB_OK;
    }
    { int wrc = mailbox_wait(env, ticket); if (wrc != BSB_OK) return wrc; }
    env->steps_done += 1;
    return report_bad_actions(env);
  }
  // Staged copies (a pageable buffer among them): actions in, bsb_step on device scratch, scalars out.  A masked step
  // also takes the mask in (and back, with budgets) and the scalars in first, so that the entries of inactive lanes
  // come back as they were; its actions are clamped and reported as on the zero-copy path.
  { int frc = drain_host_steps(env); if (frc != BSB_OK) return frc; }
  if (!env->h2d_actions) BSB_CUDA(cudaMalloc(&env->h2d_actions, B * 4));
  { int src = alloc_scalar_staging(env, host_out->reward_f64 != nullptr); if (src != BSB_OK) return src; }
  if (!device_obs && !env->d_obs) BSB_CUDA(cudaMalloc(&env->d_obs, obs_bytes));
  if (mask && !env->d_mask) BSB_CUDA(cudaMalloc(&env->d_mask, B));
  if (!mask) { int vrc = check_host_actions(env, actions, (int64_t)B); if (vrc != BSB_OK) return vrc; }
  cudaStream_t s = env->copy_stream;
  BSB_CUDA(cudaMemcpyAsync(env->h2d_actions, actions, B * 4, cudaMemcpyHostToDevice, s));
  bsb_outputs dev;
  dev.final_observation = nullptr;
  dev.observation = device_obs ? device_obs : env->d_obs;
  dev.reward = host_out->reward ? env->d_reward : nullptr;
  dev.reward_f64 = host_out->reward_f64 ? env->d_reward64 : nullptr;
  dev.discount = host_out->discount ? env->d_discount : nullptr;
  dev.step_type = host_out->step_type ? env->d_step_type : nullptr;
  const bool b2b = scalars_back_to_back(*host_out, B);
  int rc;
  if (mask) {
    BSB_CUDA(cudaMemcpyAsync(env->d_mask, mask, B, cudaMemcpyHostToDevice, s));
    if (b2b) {
      BSB_CUDA(cudaMemcpyAsync(env->d_reward, host_out->reward, 3 * B * 4, cudaMemcpyHostToDevice, s));
    } else {
      if (host_out->reward) BSB_CUDA(cudaMemcpyAsync(dev.reward, host_out->reward, B * 4, cudaMemcpyHostToDevice, s));
      if (host_out->discount) BSB_CUDA(cudaMemcpyAsync(dev.discount, host_out->discount, B * 4, cudaMemcpyHostToDevice, s));
      if (host_out->step_type) BSB_CUDA(cudaMemcpyAsync(dev.step_type, host_out->step_type, B * 4, cudaMemcpyHostToDevice, s));
    }
    if (host_out->reward_f64) BSB_CUDA(cudaMemcpyAsync(dev.reward_f64, host_out->reward_f64, B * 8, cudaMemcpyHostToDevice, s));
    rc = masked_call(env, env->h2d_actions, env->d_mask, &dev, s, MODE_STEP, 1, false, 0, nullptr, episodes_left,
                     episodes_left ? env->d_mask : nullptr);
  } else {
    rc = bsb_step(env, env->h2d_actions, &dev, s);
  }
  if (rc != BSB_OK) return rc;
  if (b2b) {
    BSB_CUDA(cudaMemcpyAsync(host_out->reward, env->d_reward, 3 * B * 4, cudaMemcpyDeviceToHost, s));
  } else {
    if (host_out->reward) BSB_CUDA(cudaMemcpyAsync(host_out->reward, dev.reward, B * 4, cudaMemcpyDeviceToHost, s));
    if (host_out->discount) BSB_CUDA(cudaMemcpyAsync(host_out->discount, dev.discount, B * 4, cudaMemcpyDeviceToHost, s));
    if (host_out->step_type) BSB_CUDA(cudaMemcpyAsync(host_out->step_type, dev.step_type, B * 4, cudaMemcpyDeviceToHost, s));
  }
  if (host_out->reward_f64) BSB_CUDA(cudaMemcpyAsync(host_out->reward_f64, dev.reward_f64, B * 8, cudaMemcpyDeviceToHost, s));
  if (host_out->observation) BSB_CUDA(cudaMemcpyAsync(host_out->observation, dev.observation, obs_bytes, cudaMemcpyDeviceToHost, s));
  if (mask && episodes_left) BSB_CUDA(cudaMemcpyAsync(mask, env->d_mask, B, cudaMemcpyDeviceToHost, s));
  BSB_CUDA(cudaStreamSynchronize(s));
  return mask ? report_bad_actions(env) : BSB_OK;
}

int32_t bsb_step_host(bsb_env* env, const int32_t* actions, const bsb_outputs* host_out, float* device_obs,
                      void* caller_stream, uint32_t flags) {
  return host_step(env, actions, nullptr, nullptr, host_out, device_obs, caller_stream, flags);
}

int32_t bsb_step_host_masked(bsb_env* env, const int32_t* actions, uint8_t* mask, int64_t* episodes_left,
                             const bsb_outputs* host_out, float* device_obs, void* caller_stream, uint32_t flags) {
  if (env && !mask) return fail(BSB_INVALID_ARGUMENT, "bsb_step_host_masked needs a mask");
  return host_step(env, actions, mask, episodes_left, host_out, device_obs, caller_stream, flags);
}


int32_t bsb_host_wait(bsb_env* env) {
  if (!env) return fail(BSB_INVALID_ARGUMENT, "null argument");
  if (env->device < 0 || !env->awaiting_ticket) return BSB_OK;
  DeviceGuard guard(env->device);
  { int rc = finish_awaited(env); if (rc != BSB_OK) return rc; }
  return report_bad_actions(env);
}

}  // extern "C"
