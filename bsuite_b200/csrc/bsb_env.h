// Internal declarations shared by the engine and the per-family translation units.
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
  // bsb_create_packed: n_settings settings of lanes_per_setting lanes each (p.pack holds their values); an ordinary
  // handle has packed = false, n_settings = 1, lanes_per_setting = batch
  bool packed;
  int32_t n_settings;
  int64_t lanes_per_setting;
  int64_t steps_done;     // step() calls so far (host counter; frozen at the switch to graph-safe mode)
  // Graph-safe mode: entered for good when a launch of this handle is first captured into a CUDA graph.  From
  // then on the device clock counts the steps (kernel comment in bsb_kernels.cuh) and steps = steps_done + clock[0].
  bool graph_safe;
  unsigned long long* clock;         // device, CLOCK_WORDS words: step count (replicated), chunk counter, finished-CTA counters
  double* sum_scratch;               // device: bsb_sum_episode_stats partials [64][5] + the ticket
  // tuning knobs (environment variables, read once per handle)
  int block_threads;      // CTA size of the transition kernel (32 / 64 / 128)
  int emit_bulk;          // TMA bulk stores for the row / board emitters
  int deep_sea_bulk;      // TMA bulk stores for deep_sea tiles (else 16-byte streaming stores)
  int deep_sea_group;     // lanes per deep_sea bulk store (0 = automatic)
  unsigned long long* work_counter;  // device counter of the dynamic chunk scheduler
  unsigned long long work_base;      // its value when the next launch starts
  int use_pdl;            // programmatic dependent launch between consecutive steps
  int graph_pdl;          // ... also between launches captured into a CUDA graph (programmatic graph edges)
  int zero_copy;          // bsb_step_host: kernel reads/writes pinned host buffers directly
  int image_stages;       // mnist TMA path: staging buffers per warp (1 or 2)
  int image_group;        // mnist TMA path: tiles per staged store (1, 2 or 4)
  int chunk_lanes;        // lanes per chunk: 0 = automatic (32; 16 / 8 for small mnist batches), BSB_CHUNK_LANES forces
  int num_sms;
  bsb::InfoNames names;
  std::vector<void*> allocs;
  std::vector<std::pair<void*, size_t> > state_blocks;  // snapshot layout
  // bsb_step_host scratch (device)
  int32_t* h2d_actions; float* d_reward; double* d_reward64; float* d_discount; int32_t* d_step_type; float* d_obs;
  cudaStream_t copy_stream;
  cudaEvent_t order_event;            // BSB_HOST_ORDER_AFTER_STREAM: fences copy_stream behind the caller's stream
  cudaEvent_t fence_event;            // BSB_HOST_FENCE_CALLER: fences the caller's stream behind a two-phase host step
  // Out-of-range actions (ADVICE r01): the kernels clamp them before any table index or state packing and raise
  // this pinned flag; bsb_step_host / bsb_invalid_actions report it.
  int32_t* bad_action_host; int32_t* bad_action_dev;
  // Host-driven steps without a stream synchronise (bsb_step_host on pinned buffers): the kernel signals completion
  // through a pinned mailbox the host spins on; with BSB_HOST_PRELAUNCH the next step's kernel is already queued
  // and waits for the mailbox doorbell (bsb_kernels.cuh, HostMailbox).
  bsb::HostMailbox* mailbox; bsb::HostMailbox* mailbox_dev; bsb::DeviceMail* mail;
  unsigned long long next_ticket;     // last ticket handed out
  unsigned long long awaiting_ticket; // a BSB_HOST_NO_WAIT step whose completion word has not been collected yet (0 = none)
  unsigned long long pending_ticket;  // pre-launched launch waiting for its doorbell (0 = none); it is for step steps_done
  unsigned long long doorbell_timeout_ns;
  int host_spin;                      // BSB_HOST_SPIN (default 1): completion through the mailbox instead of a synchronise
  int host_split;                     // BSB_HOST_SPLIT (default 1): BSB_HOST_NO_WAIT two-phase steps run as two launches (transitions, observations)
  int host_early;                     // BSB_HOST_EARLY (default 1): two-phase host steps (scalars first) where the family allows
  bool early_inflight;                // a two-phase host step may still be streaming observations on copy_stream
  int host_stage_actions;             // BSB_HOST_STAGE_ACTIONS (default 1): two-phase steps get their actions by DMA on a side stream instead of reading them in place
  cudaStream_t h2d_stream; cudaEvent_t h2d_event;
};

namespace bsb {
// One entry per family, each defined in its own translation unit (fam_<name>.cu).
// deep_sea and catch also run the two-phase host step (`two_phase`: its arguments).  Each also reaches its same-step
// (ss_<name>.cu), reduced-dtype (obs_<name>.cu) and, but deep_sea, packed (pk_<name>.cu) instantiations.
int run_deep_sea(bsb_env*, const LaunchArgs&, cudaStream_t, const TwoPhaseArgs* two_phase = nullptr);
int run_catch(bsb_env*, const LaunchArgs&, cudaStream_t, const TwoPhaseArgs* two_phase = nullptr);
int run_cartpole(bsb_env*, const LaunchArgs&, cudaStream_t);
int run_cartpole_swingup(bsb_env*, const LaunchArgs&, cudaStream_t);
int run_mountain_car(bsb_env*, const LaunchArgs&, cudaStream_t);
int run_memory_chain(bsb_env*, const LaunchArgs&, cudaStream_t);
int run_bandit(bsb_env*, const LaunchArgs&, cudaStream_t);
int run_umbrella_chain(bsb_env*, const LaunchArgs&, cudaStream_t);
int run_discounting_chain(bsb_env*, const LaunchArgs&, cudaStream_t);
int run_mnist(bsb_env*, const LaunchArgs&, cudaStream_t);
}  // namespace bsb
