// Internal declarations shared by the engine and the kernel-variant translation units.
#pragma once
#include <cuda_runtime.h>

#include <atomic>
#include <string>
#include <utility>
#include <vector>

#include "../../include/bsuite_b200.h"
#include "bsb_kernels.cuh"

namespace bsb {

struct InfoNames { int n; const char* names[BSB_MAX_INFO]; };

int fail(int code, const std::string& msg);           // records the thread-local error string
const char* last_error_cstr();
extern std::atomic<int64_t> g_launches;                // kernels launched by this library
bool in_compressed_block(const void* p);               // p lies in a compressed bsb_obs_malloc block (bsb_memory.cu)
}  // namespace bsb
struct bsb_env;
namespace bsb {
int drain_log_rows(bsb_env* e);                         // waits out host steps in flight, as bsb_read_log_rows does

// Kernels and host path of kernel variant V (bsb_dispatch.cuh), explicitly instantiated for each entry of the variant
// list (BSB_VARIANTS) in the translation unit the list gives it (bsb_variants.cu).  `two_phase`: a two-phase host step.
template <class V> int run_variant(bsb_env*, const LaunchArgs&, cudaStream_t, const TwoPhaseArgs* two_phase);
// Masked calls of variant V (bsb_reset_masked / bsb_step_masked / bsb_rollout_masked / bsb_step_host_masked /
// bsb_advance_masked / bsb_step_budgeted): `mask` [B] and `episodes_left` [B] (nullable) live where the handle's
// state does, or `mask` is a pinned host buffer's device alias.  `mask_out` (masked host steps with budgets and
// budgeted steps, else null): where spent lanes' mask bytes are cleared.  `previous` (budgeted steps, else null): the
// outputs that receive the masked-in lanes' current entries before the step.  `policy` (bsb_step_budgeted_policy,
// else null): the rule that chooses a budgeted step's actions.  `replay` (bsb_step_budgeted_record, else null): the
// lanes' rings a budgeted step appends its transitions to.  `sequence` (bsb_step_budgeted_sequence, else null): the
// lanes' sequence buffers a budgeted step appends its transitions to.  `ensemble` (bsb_step_budgeted_ensemble, else
// null): the heads and values of an ensemble step, whose `policy` is then its epsilon-greedy rule.
template <class V> int run_masked(bsb_env*, const LaunchArgs&, const uint8_t* mask, int64_t* episodes_left,
                                  uint8_t* mask_out, const bsb_outputs* previous, const bsb_policy* policy,
                                  const bsb_replay* replay, const bsb_sequence* sequence,
                                  const bsb_ensemble_policy* ensemble, cudaStream_t);
// An entry of the variant list, as bsb_create looks it up (bsb_engine.cu).
struct VariantEntry {
  int family, obs_dtype, mode;
  bool mt, two_phase;
  int (*run)(bsb_env*, const LaunchArgs&, cudaStream_t, const TwoPhaseArgs*);
  int (*run_masked)(bsb_env*, const LaunchArgs&, const uint8_t*, int64_t*, uint8_t*, const bsb_outputs*, const bsb_policy*,
                    const bsb_replay*, const bsb_sequence*, const bsb_ensemble_policy*, cudaStream_t);
};

#define BSB_CUDA(expr)                                                                   \
  do {                                                                                   \
    cudaError_t e__ = (expr);                                                            \
    if (e__ != cudaSuccess)                                                              \
      return ::bsb::fail(e__ == cudaErrorMemoryAllocation ? BSB_OUT_OF_MEMORY : BSB_CUDA_ERROR, \
                         std::string(#expr) + ": " + cudaGetErrorString(e__));           \
  } while (0)

}  // namespace bsb

struct bsb_env {
  bsb::EnvParams p;
  int device;             // BSB_DEVICE_HOST or CUDA ordinal
  int obs_dtype;          // bsb_obs_dtype of the observations this handle writes
  int obs_elem_bytes;     // ... and their size: 4, 2 or 1
  bool same_step;         // BSB_FLAG_SAME_STEP_RESET: a LAST lane is reset in the same call
  const bsb::VariantEntry* variant;   // the compiled variant of the handle's family, obs_dtype and mode: its runner
  // bsb_create_packed: n_settings settings of lanes_per_setting lanes each (p.pack holds their values); an ordinary
  // handle has packed = false, n_settings = 1, lanes_per_setting = batch
  bool packed;
  int32_t n_settings;
  int64_t lanes_per_setting;
  // bsb_create_ragged (packed is true as well): setting k's observations are a dense [lanes_per_setting, rows, cols]
  // block at element obs_offset[k] of each step of step_elems elements; group_lanes[k] is the deep_sea bulk path's
  // lanes per store (0: none).  Every other handle: one block per setting of lanes_per_setting * p.obs_numel elements.
  bool ragged;
  std::vector<int64_t> obs_offset;
  std::vector<int32_t> obs_rows, obs_cols, group_lanes;
  int64_t step_elems;
  int64_t steps_done;     // step() calls so far (host counter; frozen at the switch to graph-safe mode)
  // Graph-safe mode: entered for good when a launch of this handle is first captured into a CUDA graph.  From
  // then on the device clock counts the steps (kernel comment in bsb_kernels.cuh) and steps = steps_done + clock[0].
  bool graph_safe;
  unsigned long long* clock;         // device, CLOCK_WORDS words: step count (replicated), chunk counter, finished-CTA counters
  double* sum_scratch;               // device: per setting, the sum kernel's partials [64][5] + the ticket
  unsigned long long* work_counter;  // device counter of the dynamic chunk scheduler
  unsigned long long work_base;      // its value when the next launch starts
  int num_sms;
  bsb::InfoNames names;
  std::vector<void*> allocs;
  std::vector<std::pair<void*, size_t> > state_blocks;  // snapshot layout
  // bsb_step_host scratch (device)
  int32_t* h2d_actions; float* d_reward; double* d_reward64; float* d_discount; int32_t* d_step_type; float* d_obs;
  uint8_t* d_mask;                    // bsb_step_host_masked on a pageable mask: its device staging
  cudaStream_t copy_stream;
  cudaEvent_t order_event;            // BSB_HOST_ORDER_AFTER_STREAM: fences copy_stream behind the caller's stream
  cudaEvent_t fence_event;            // BSB_HOST_FENCE_CALLER: fences the caller's stream behind a two-phase host step
  // Out-of-range actions (ADVICE r01): the kernels clamp them before any table index or state packing and raise
  // this pinned flag; bsb_step_host / bsb_invalid_actions report it.  A host handle's flag is bad_action_flag, which
  // only bsb_step_budgeted_policy raises (for invalid value rows): its actions are validated before anything moves.
  int32_t* bad_action_host; int32_t* bad_action_dev;
  int32_t bad_action_flag;
  // Host-driven steps without a stream synchronise (bsb_step_host on pinned buffers): the kernel signals completion
  // through a pinned mailbox the host spins on (bsb_kernels.cuh, HostMailbox).
  bsb::HostMailbox* mailbox; bsb::HostMailbox* mailbox_dev; bsb::DeviceMail* mail;
  unsigned long long next_ticket;     // last ticket handed out
  unsigned long long awaiting_ticket; // a BSB_HOST_NO_WAIT step whose completion word has not been collected yet (0 = none)
  bool early_inflight;                // a two-phase host step may still be streaming observations on copy_stream
  cudaStream_t h2d_stream; cudaEvent_t h2d_event;     // two-phase host steps: the actions' DMA on a side stream
};

