// Interpolating branch of ImageObservation / to_image (utils/wrappers.py:207-219): every [h, w] observation plane
// of a batch becomes skimage.transform.resize(plane, (H, W), preserve_range=True) broadcast over C trailing floats.
//
// skimage (>= 0.19) builds resize on scipy.ndimage; restated operation by operation (oracle/image_oracle.py is the
// same computation written as the scipy calls):
//   1. anti-aliasing, only when H < h or W < w: gaussian_filter(mode='mirror') per axis with sigma > 0, rows first.
//      scipy's correlate1d sums a symmetric kernel as centre * tap[0], then (left + right) * tap[j] from the
//      farthest tap inwards, in float64; each pass is rounded to float32.
//   2. zoom(order=1, mode='mirror', grid_mode=True): sum over the 2 x 2 neighbourhood, row-major, from 0.0, of
//      (value * row_weight) * col_weight in float64, rounded to float32.
//   3. np.clip to [min, max] of the unfiltered plane.
// The index / weight tables and the Gaussian taps come from the caller (bsuite_b200/imaging.py builds them with
// numpy, with the operations scipy uses), so the arithmetic here is only the sums above; the build passes
// --fmad=false, so no product is contracted into an fma.
//
// The hot path is HBM writes: one (84, 84, 4) image is 112 896 bytes, far more than the plane it comes from.  A CTA
// takes one lane at a time (persistent grid): the plane is staged in shared memory (and filtered there), the output
// is rendered in 16 KB chunks into two alternating shared-memory stages, and each chunk leaves with one TMA bulk
// store carrying the evict_first L2 hint, as the observation emitters do.  A chunk whose global address is not
// 16-byte aligned leaves with 16-byte streaming stores instead (scalar head and tail).  Planes too large for the
// stage are read from global memory, and filtered into a per-CTA scratch the plan owns.
#include <cstring>
#include <vector>

#include "bsb_env.h"

namespace bsb {
namespace {

struct ImageParams {
  int32_t h, w, H, W, C, ry, rx;
  const int32_t* row_index; const double* row_weight;   // [H][2]
  const int32_t* col_index; const double* col_weight;   // [W][2]
  const double* row_taps; const double* col_taps;       // [radius + 1]: centre, distance 1 .. radius
};

static const int IMG_THREADS = 256;
static const int OUT_STAGE_FLOATS = 4096;               // one output chunk (16 KB); two stages per CTA
static const int PLANE_STAGE_FLOATS = 12288;            // input plane (+ its filtered copy) staged in shared memory
static const size_t SCRATCH_BYTES_MAX = 256u << 20;     // global scratch of the unstaged, filtered path

// scipy's 'mirror' extension of an integer index: period 2n - 2, a length-1 axis maps everything to 0.
BSB_HD int mirror_index(int i, int n) {
  if (n == 1) return 0;
  const int period = 2 * n - 2;
  i = (i < 0 ? -i : i) % period;
  return i >= n ? period - i : i;
}

// Running min / max of skimage's clip (_clip_warp_output): NaN values are skipped (np.nanmin / np.nanmax when the
// plane holds a NaN, which equal np.min / np.max otherwise); the result is NaN only when every value is.
BSB_HD float nan_min(float acc, float v) { return (v != v) ? acc : ((acc != acc || v < acc) ? v : acc); }
BSB_HD float nan_max(float acc, float v) { return (v != v) ? acc : ((acc != acc || v > acc) ? v : acc); }

// One output element of a Gaussian pass along rows (axis 0) or columns (axis 1), rounded to float32.
BSB_HD float gauss_pass(const float* src, int h, int w, int y, int x, const double* taps, int r, bool along_rows) {
  double t = (double)src[y * w + x] * taps[0];
  for (int j = r; j >= 1; --j) {
    const double left = along_rows ? (double)src[mirror_index(y - j, h) * w + x] : (double)src[y * w + mirror_index(x - j, w)];
    const double right = along_rows ? (double)src[mirror_index(y + j, h) * w + x] : (double)src[y * w + mirror_index(x + j, w)];
    t += (left + right) * taps[j];
  }
  return (float)t;
}

// Order-1 zoom of output pixel (oy, ox), clipped to [lo, hi].
BSB_HD float image_pixel(const float* plane, const ImageParams& p, int oy, int ox, float lo, float hi) {
  const int y0 = p.row_index[2 * oy], y1 = p.row_index[2 * oy + 1];
  const int x0 = p.col_index[2 * ox], x1 = p.col_index[2 * ox + 1];
  const double wy0 = p.row_weight[2 * oy], wy1 = p.row_weight[2 * oy + 1];
  const double wx0 = p.col_weight[2 * ox], wx1 = p.col_weight[2 * ox + 1];
  double t = 0.0;
  t += (double)plane[y0 * p.w + x0] * wy0 * wx0;
  t += (double)plane[y0 * p.w + x1] * wy0 * wx1;
  t += (double)plane[y1 * p.w + x0] * wy1 * wx0;
  t += (double)plane[y1 * p.w + x1] * wy1 * wx1;
  const float v = (float)t;
  if (lo != lo) return lo;                               // an all-NaN plane: np.clip against NaN bounds is NaN
  return v < lo ? lo : (v > hi ? hi : v);                // np.clip(v, lo, hi) = minimum(maximum(v, lo), hi)
}

// Host path: the same functions, lane by lane.
void host_to_image(const ImageParams& p, const float* in, int64_t batch, float* out) {
  const int n = p.h * p.w;
  const int64_t N = (int64_t)p.H * p.W * p.C;
  std::vector<float> b1((size_t)n), b2((size_t)n);
  for (int64_t lane = 0; lane < batch; ++lane) {
    const float* src = in + lane * n;
    float lo = src[0], hi = src[0];
    for (int i = 1; i < n; ++i) { lo = nan_min(lo, src[i]); hi = nan_max(hi, src[i]); }
    const float* plane = src;
    if (p.ry > 0) {
      for (int y = 0; y < p.h; ++y) for (int x = 0; x < p.w; ++x) b1[y * p.w + x] = gauss_pass(plane, p.h, p.w, y, x, p.row_taps, p.ry, true);
      plane = b1.data();
    }
    if (p.rx > 0) {
      float* dst = plane == b1.data() ? b2.data() : b1.data();
      for (int y = 0; y < p.h; ++y) for (int x = 0; x < p.w; ++x) dst[y * p.w + x] = gauss_pass(plane, p.h, p.w, y, x, p.col_taps, p.rx, false);
      plane = dst;
    }
    float* dst = out + lane * N;
    for (int oy = 0; oy < p.H; ++oy)
      for (int ox = 0; ox < p.W; ++ox) {
        const float v = image_pixel(plane, p, oy, ox, lo, hi);
        for (int c = 0; c < p.C; ++c) *dst++ = v;
      }
  }
}

// staged: the plane (and, when filtered, its filtered copy) lives in shared memory after the two output stages;
// otherwise it is read from `in` and filtered into scratch[blockIdx.x][2][h * w], which is why launches of such a
// plan must not overlap (include/bsuite_b200.h).
__global__ void __launch_bounds__(IMG_THREADS) to_image_kernel(const ImageParams p, const float* __restrict__ in,
                                                                int64_t batch, float* __restrict__ out, float* scratch,
                                                                int staged) {
  extern __shared__ float4 smem_raw[];
  __shared__ float red_lo[IMG_THREADS / 32], red_hi[IMG_THREADS / 32];
  float* const stages = reinterpret_cast<float*>(smem_raw);
  float* const plane_stage = stages + 2 * OUT_STAGE_FLOATS;
  const int n = p.h * p.w;
  const int N = p.H * p.W * p.C;                        // floats per lane (< 2^31, checked by the plan)
  const int tid = threadIdx.x;
  unsigned chunk_no = 0;
  for (int64_t lane = blockIdx.x; lane < batch; lane += gridDim.x) {
    const float* src = in + lane * n;
    const float* orig;
    float *b1, *b2;
    if (staged) {
      for (int i = tid; i < n; i += IMG_THREADS) plane_stage[i] = __ldg(src + i);
      orig = plane_stage; b1 = plane_stage + n; b2 = plane_stage;     // the column pass may overwrite the original
      __syncthreads();
    } else {
      orig = src; b1 = scratch + (size_t)blockIdx.x * 2 * (size_t)n; b2 = b1 + n;
    }
    // [min, max] of the unfiltered plane
    float lo = orig[0], hi = orig[0];
    for (int i = tid; i < n; i += IMG_THREADS) { const float v = orig[i]; lo = nan_min(lo, v); hi = nan_max(hi, v); }
    for (int s = 16; s >= 1; s >>= 1) {
      lo = nan_min(lo, __shfl_xor_sync(0xffffffffu, lo, s));
      hi = nan_max(hi, __shfl_xor_sync(0xffffffffu, hi, s));
    }
    if ((tid & 31) == 0) { red_lo[tid >> 5] = lo; red_hi[tid >> 5] = hi; }
    __syncthreads();
    for (int k = 0; k < IMG_THREADS / 32; ++k) { lo = nan_min(lo, red_lo[k]); hi = nan_max(hi, red_hi[k]); }
    // anti-aliasing passes (each rounded to float32)
    const float* plane = orig;
    if (p.ry > 0) {
      for (int i = tid; i < n; i += IMG_THREADS) b1[i] = gauss_pass(plane, p.h, p.w, i / p.w, i % p.w, p.row_taps, p.ry, true);
      __syncthreads();
      plane = b1;
    }
    if (p.rx > 0) {
      float* dst = plane == b1 ? b2 : b1;
      for (int i = tid; i < n; i += IMG_THREADS) dst[i] = gauss_pass(plane, p.h, p.w, i / p.w, i % p.w, p.col_taps, p.rx, false);
      __syncthreads();
      plane = dst;
    }
    // render and ship the lane's N contiguous floats in chunks
    float* const lane_out = out + lane * (int64_t)N;
    for (int f0 = 0; f0 < N; f0 += OUT_STAGE_FLOATS, ++chunk_no) {
      const int len = min(OUT_STAGE_FLOATS, N - f0);
      float* const buf = stages + (chunk_no & 1u) * OUT_STAGE_FLOATS;
      if (tid == 0) bulk_wait_read<1>();                // the group of two chunks ago (this stage) has been read
      __syncthreads();
      for (int q = tid * 4; q < len; q += IMG_THREADS * 4) {
        // four consecutive floats; a pixel is evaluated once and repeated over its C channels in registers
        const int e = f0 + q, m = min(4, len - q);
        int pix = e / p.C, next = (pix + 1) * p.C;
        float v = image_pixel(plane, p, pix / p.W, pix % p.W, lo, hi);
        float r[4] = {v, v, v, v};
        for (int k = 1; k < m; ++k) {
          if (e + k >= next) { pix = (e + k) / p.C; next = (pix + 1) * p.C; v = image_pixel(plane, p, pix / p.W, pix % p.W, lo, hi); }
          r[k] = v;
        }
        if (m == 4) *reinterpret_cast<float4*>(buf + q) = make_float4(r[0], r[1], r[2], r[3]);
        else for (int k = 0; k < m; ++k) buf[q + k] = r[k];
      }
      fence_proxy_async_smem();
      __syncthreads();
      float* const g = lane_out + f0;
      const unsigned mis = (unsigned)(reinterpret_cast<uintptr_t>(g) & 15u);
      if (mis == 0) {
        const int body = len & ~3;
        if (tid == 0 && body > 0) bulk_store_obs(g, buf, (uint32_t)body * 4u);
        if (tid < len - body) st_stream(g + body + tid, buf[body + tid]);
      } else {                                          // 16-byte streaming stores between a scalar head and tail
        const int head = min(len, (int)((16u - mis) >> 2));
        const int body4 = (len - head) >> 2, tail = head + 4 * body4;
        if (tid < head) st_stream(g + tid, buf[tid]);
        for (int i = tid; i < body4; i += IMG_THREADS) {
          const float* s = buf + head + 4 * i;
          st_stream(reinterpret_cast<float4*>(g + head) + i, make_float4(s[0], s[1], s[2], s[3]));
        }
        if (tid < len - tail) st_stream(g + tail + tid, buf[tail + tid]);
      }
      // One bulk group per chunk, empty when the chunk left without a bulk store: the wait_group.read 1 above then
      // always covers the store that last read the stage about to be rewritten.
      if (tid == 0) bulk_commit();
    }
  }
  if (tid == 0) bulk_wait_all();
}

struct DeviceGuard {
  int prev; bool on;
  explicit DeviceGuard(int dev) : prev(0), on(dev >= 0) { if (on) { cudaGetDevice(&prev); cudaSetDevice(dev); } }
  ~DeviceGuard() { if (on) cudaSetDevice(prev); }
};

}  // namespace
}  // namespace bsb

struct bsb_image_plan {
  int device;
  bsb::ImageParams p;
  void* tables;            // row_index, col_index, row_weight, col_weight, row_taps, col_taps (device or host)
  float* scratch;          // device, unstaged filtered path only
  int staged;              // the plane fits the shared-memory stage
  size_t smem_bytes;
  int max_ctas;            // persistent grid of a launch (fewer when the batch is smaller)
};

using bsb::fail;

namespace {

void destroy_plan(bsb_image_plan* plan) {
  if (plan->device >= 0) {
    bsb::DeviceGuard guard(plan->device);
    if (plan->tables) cudaFree(plan->tables);
    if (plan->scratch) cudaFree(plan->scratch);
  } else {
    free(plan->tables);
  }
  delete plan;
}

int check_table(const void* ptr, int64_t len, int64_t want, const char* name) {
  if (len != want) return fail(BSB_INVALID_ARGUMENT, std::string(name) + " has " + std::to_string(len) +
                                                         " elements, expected " + std::to_string(want));
  if (want > 0 && !ptr) return fail(BSB_INVALID_ARGUMENT, std::string(name) + " is null");
  return BSB_OK;
}

}  // namespace

extern "C" {

int32_t bsb_image_plan_create(const bsb_image_desc* desc, int32_t device, bsb_image_plan** out) {
  if (!desc || !out) return fail(BSB_INVALID_ARGUMENT, "null argument");
  *out = nullptr;
  const bsb_image_desc& d = *desc;
  if (d.in_rows < 1 || d.in_cols < 1 || d.out_rows < 1 || d.out_cols < 1)
    return fail(BSB_INVALID_ARGUMENT, "image dims must be >= 1");
  if (d.channels < 1) return fail(BSB_INVALID_ARGUMENT, "channels must be >= 1");
  if (d.row_radius < 0 || d.col_radius < 0) return fail(BSB_INVALID_ARGUMENT, "Gaussian radius must be >= 0");
  if (d.row_radius > (1 << 20) || d.col_radius > (1 << 20)) return fail(BSB_UNSUPPORTED, "Gaussian radius above 2^20");
  if ((int64_t)d.in_rows * d.in_cols > (1ll << 30)) return fail(BSB_UNSUPPORTED, "input plane above 2^30 values");
  if ((int64_t)d.out_rows * d.out_cols * d.channels >= (1ll << 31) - bsb::OUT_STAGE_FLOATS)
    return fail(BSB_UNSUPPORTED, "output image above 2^31 floats");
  int rc;
  if ((rc = check_table(d.row_index, d.row_index_len, 2ll * d.out_rows, "row_index")) != BSB_OK) return rc;
  if ((rc = check_table(d.row_weight, d.row_weight_len, 2ll * d.out_rows, "row_weight")) != BSB_OK) return rc;
  if ((rc = check_table(d.col_index, d.col_index_len, 2ll * d.out_cols, "col_index")) != BSB_OK) return rc;
  if ((rc = check_table(d.col_weight, d.col_weight_len, 2ll * d.out_cols, "col_weight")) != BSB_OK) return rc;
  if ((rc = check_table(d.row_taps, d.row_taps_len, d.row_radius ? d.row_radius + 1 : 0, "row_taps")) != BSB_OK) return rc;
  if ((rc = check_table(d.col_taps, d.col_taps_len, d.col_radius ? d.col_radius + 1 : 0, "col_taps")) != BSB_OK) return rc;
  for (int64_t k = 0; k < 2ll * d.out_rows; ++k)
    if (d.row_index[k] < 0 || d.row_index[k] >= d.in_rows) return fail(BSB_INVALID_ARGUMENT, "row_index entry outside [0, in_rows)");
  for (int64_t k = 0; k < 2ll * d.out_cols; ++k)
    if (d.col_index[k] < 0 || d.col_index[k] >= d.in_cols) return fail(BSB_INVALID_ARGUMENT, "col_index entry outside [0, in_cols)");
  int num_sms = 132;
  if (device >= 0) {
    int count = 0;
    cudaError_t err = cudaGetDeviceCount(&count);
    if (err != cudaSuccess || count <= 0)
      return fail(BSB_CUDA_ERROR, std::string("no CUDA device available (") + cudaGetErrorString(err) +
                                      "); this engine has no implicit CPU fallback -- pass device=BSB_DEVICE_HOST explicitly for the host path");
    if (device >= count) return fail(BSB_INVALID_ARGUMENT, "device ordinal out of range");
    int sms = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) == cudaSuccess && sms > 0) num_sms = sms;
  } else if (device != BSB_DEVICE_HOST) {
    return fail(BSB_INVALID_ARGUMENT, "device must be >= 0 or BSB_DEVICE_HOST");
  }

  // one block: int32 indices first, then float64 weights and taps (8-byte aligned)
  const size_t H = (size_t)d.out_rows, W = (size_t)d.out_cols;
  const size_t n_idx = 2 * H + 2 * W + ((2 * H + 2 * W) & 1);
  const size_t ry = d.row_radius ? (size_t)d.row_radius + 1 : 0, rx = d.col_radius ? (size_t)d.col_radius + 1 : 0;
  const size_t bytes = n_idx * 4 + (2 * H + 2 * W + ry + rx) * 8;
  std::vector<unsigned char> host(bytes, 0);
  int32_t* idx = reinterpret_cast<int32_t*>(host.data());
  double* dbl = reinterpret_cast<double*>(host.data() + n_idx * 4);
  memcpy(idx, d.row_index, 2 * H * 4);
  memcpy(idx + 2 * H, d.col_index, 2 * W * 4);
  memcpy(dbl, d.row_weight, 2 * H * 8);
  memcpy(dbl + 2 * H, d.col_weight, 2 * W * 8);
  if (ry) memcpy(dbl + 2 * H + 2 * W, d.row_taps, ry * 8);
  if (rx) memcpy(dbl + 2 * H + 2 * W + ry, d.col_taps, rx * 8);

  bsb_image_plan* plan = new bsb_image_plan();
  plan->device = device; plan->tables = nullptr; plan->scratch = nullptr;
  bsb::DeviceGuard guard(device);
  if (device >= 0) {
    cudaError_t err = cudaMalloc(&plan->tables, bytes);
    if (err == cudaSuccess) err = cudaMemcpy(plan->tables, host.data(), bytes, cudaMemcpyHostToDevice);
    if (err != cudaSuccess) { destroy_plan(plan); return fail(err == cudaErrorMemoryAllocation ? BSB_OUT_OF_MEMORY : BSB_CUDA_ERROR, std::string("image tables: ") + cudaGetErrorString(err)); }
  } else {
    plan->tables = malloc(bytes);
    if (!plan->tables) { destroy_plan(plan); return fail(BSB_OUT_OF_MEMORY, "malloc failed"); }
    memcpy(plan->tables, host.data(), bytes);
  }
  const unsigned char* base = static_cast<const unsigned char*>(plan->tables);
  const int32_t* t_idx = reinterpret_cast<const int32_t*>(base);
  const double* t_dbl = reinterpret_cast<const double*>(base + n_idx * 4);
  bsb::ImageParams& p = plan->p;
  p.h = d.in_rows; p.w = d.in_cols; p.H = d.out_rows; p.W = d.out_cols; p.C = d.channels;
  p.ry = d.row_radius; p.rx = d.col_radius;
  p.row_index = t_idx; p.col_index = t_idx + 2 * H;
  p.row_weight = t_dbl; p.col_weight = t_dbl + 2 * H;
  p.row_taps = ry ? t_dbl + 2 * H + 2 * W : nullptr;
  p.col_taps = rx ? t_dbl + 2 * H + 2 * W + ry : nullptr;

  const int64_t n = (int64_t)p.h * p.w;
  const bool filtered = p.ry > 0 || p.rx > 0;
  const int64_t plane_floats = filtered ? 2 * n : n;
  plan->staged = plane_floats <= bsb::PLANE_STAGE_FLOATS ? 1 : 0;
  plan->smem_bytes = (size_t)(2 * bsb::OUT_STAGE_FLOATS + (plan->staged ? plane_floats : 0)) * sizeof(float);
  plan->max_ctas = num_sms;
  if (device >= 0) {
    const int smem_max = (2 * bsb::OUT_STAGE_FLOATS + bsb::PLANE_STAGE_FLOATS) * (int)sizeof(float);
    cudaError_t err = cudaFuncSetAttribute(bsb::to_image_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max);
    int per_sm = 0;
    if (err == cudaSuccess)
      err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, bsb::to_image_kernel, bsb::IMG_THREADS, plan->smem_bytes);
    if (err != cudaSuccess) { destroy_plan(plan); return fail(BSB_CUDA_ERROR, std::string("image kernel: ") + cudaGetErrorString(err)); }
    plan->max_ctas = num_sms * (per_sm > 0 ? per_sm : 1);
    if (!plan->staged && filtered) {                     // per-CTA scratch: the row-filtered and the filtered plane
      const size_t per_cta = (size_t)(2 * n) * sizeof(float);
      const size_t fit = bsb::SCRATCH_BYTES_MAX / per_cta;
      if ((size_t)plan->max_ctas > fit) plan->max_ctas = fit > 0 ? (int)fit : 1;
      err = cudaMalloc(&plan->scratch, per_cta * (size_t)plan->max_ctas);
      if (err != cudaSuccess) { destroy_plan(plan); return fail(err == cudaErrorMemoryAllocation ? BSB_OUT_OF_MEMORY : BSB_CUDA_ERROR, std::string("image scratch: ") + cudaGetErrorString(err)); }
    }
  }
  *out = plan;
  return BSB_OK;
}

int32_t bsb_image_plan_destroy(bsb_image_plan* plan) { if (plan) destroy_plan(plan); return BSB_OK; }

int32_t bsb_to_image(bsb_image_plan* plan, const float* in, int64_t batch, float* out, void* stream) {
  if (!plan) return fail(BSB_INVALID_ARGUMENT, "null plan");
  if (batch < 0) return fail(BSB_INVALID_ARGUMENT, "batch must be >= 0");
  if (batch == 0) return BSB_OK;
  if (!in || !out) return fail(BSB_INVALID_ARGUMENT, "null in / out");
  if ((reinterpret_cast<uintptr_t>(in) & 3u) || (reinterpret_cast<uintptr_t>(out) & 3u))
    return fail(BSB_INVALID_ARGUMENT, "in / out must be 4-byte aligned float32 arrays");
  if (plan->device < 0) {
    bsb::host_to_image(plan->p, in, batch, out);
    return BSB_OK;
  }
  bsb::DeviceGuard guard(plan->device);
  const int grid = (int)(batch < (int64_t)plan->max_ctas ? batch : (int64_t)plan->max_ctas);
  bsb::to_image_kernel<<<grid, bsb::IMG_THREADS, plan->smem_bytes, static_cast<cudaStream_t>(stream)>>>(
      plan->p, in, batch, out, plan->scratch, plan->staged);
  bsb::g_launches.fetch_add(1);
  BSB_CUDA(cudaGetLastError());
  return BSB_OK;
}

}  // extern "C"
