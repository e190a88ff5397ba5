// Per-lane random streams: a bit source (Philox4x64-10 or MT19937) under
// numpy's *legacy* RandomState distribution algorithms.
//
// The reference draws every random number from numpy.random.RandomState
// (deep_sea.py:77, catch.py:58, cartpole.py:91, mountain_car.py:55,
// memory_chain.py:45, umbrella_chain.py:52, mnist.py:53, wrappers.py:267,330).
// numpy is a third-party dependency of the reference (setup.py:85, unpinned;
// 2.3.5 in this image); the algorithms restated here are the ones SURVEY.md 8a
// "RNG draw table" lists:
//   rand()            next_double of the bit generator
//   uniform(lo, hi)   lo + (hi - lo) * next_double
//   binomial(1, .5)   inversion, which for n=1, p=.5 reduces to (u > 0.5)
//   randint(n)        masked rejection on next_uint32; randint(1) draws nothing
//   randn()           Marsaglia polar with the second variate cached
// Parity of these restatements is pinned by tests against numpy itself.
#pragma once
#include <stdint.h>
#include <math.h>

#if defined(__CUDACC__)
#define BSB_HD __host__ __device__ __forceinline__
#else
#define BSB_HD inline
#endif

namespace bsb {

typedef uint64_t u64;
typedef uint32_t u32;

BSB_HD u64 mulhi64(u64 a, u64 b) {
#if defined(__CUDA_ARCH__)
  return __umul64hi(a, b);
#else
  return (u64)(((unsigned __int128)a * (unsigned __int128)b) >> 64);
#endif
}

// ---------------------------------------------------------------------------
// Philox4x64-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3",
// SC'11), with the constants and word order of numpy.random.Philox.
// ---------------------------------------------------------------------------
struct PhiloxBlock { u64 v0, v1, v2, v3; };

BSB_HD PhiloxBlock philox4x64_10(u64 c0, u64 c1, u64 c2, u64 c3, u64 k0, u64 k1) {
  const u64 M0 = 0xD2E7470EE14C6C93ull, M1 = 0xCA5A826395121157ull;
  const u64 W0 = 0x9E3779B97F4A7C15ull, W1 = 0xBB67AE8584CAA73Bull;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
  for (int r = 0; r < 10; ++r) {
    const u64 hi0 = mulhi64(M0, c0), lo0 = M0 * c0;
    const u64 hi1 = mulhi64(M1, c2), lo1 = M1 * c2;
    const u64 n0 = hi1 ^ c1 ^ k0;
    const u64 n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += W0; k1 += W1;
  }
  PhiloxBlock b; b.v0 = c0; b.v1 = c1; b.v2 = c2; b.v3 = c3;
  return b;
}

// Stream ids carried in counter word 3.
enum : u64 { STREAM_ENV = 0, STREAM_WRAPPER = 1, STREAM_ACTIONS = 2, STREAM_POLICY = 3, STREAM_REPLAY = 4,
             STREAM_HEAD = 5, STREAM_BOOTSTRAP = 6 };

// On-device uniform random actions (the workload of baselines/random/agent.py:35-37).
// The action stream of a lane is the Philox stream (key = (action_seed, global lane), counter word 3 =
// STREAM_ACTIONS) read as 32-bit chunks: step s uses chunk (s & 7) of block (s >> 3); a chunk r maps to
// floor(r * n / 2^32) (multiply-shift, no rejection).  One block serves 8 consecutive steps of a lane.
struct ActionStream {
  u64 blk_index;          // block currently cached (~0 = none)
  PhiloxBlock blk;
  BSB_HD void open() { blk_index = ~0ull; blk.v0 = blk.v1 = blk.v2 = blk.v3 = 0; }
  BSB_HD int32_t sample(u64 action_seed, u64 global_lane, u64 step, int32_t n) {
    const u64 want = step >> 3;
    if (want != blk_index) { blk = philox4x64_10(want, 0, 0, STREAM_ACTIONS, action_seed, global_lane); blk_index = want; }
    const u32 c = (u32)(step & 7);
    const u64 w = (c >> 1) == 0 ? blk.v0 : ((c >> 1) == 1 ? blk.v1 : ((c >> 1) == 2 ? blk.v2 : blk.v3));
    const u32 r = (c & 1) ? (u32)(w >> 32) : (u32)w;
    return (int32_t)(((u64)r * (u64)(u32)n) >> 32);
  }
};

BSB_HD int32_t sample_action(u64 action_seed, u64 global_lane, u64 step, int32_t n) {
  ActionStream s; s.open();
  return s.sample(action_seed, global_lane, step, n);
}

// exp(x) built from + - * and ldexp alone, so the host path and the kernels (compiled with --fmad=false /
// -ffp-contract=off) compute the same bits, which libm's and libdevice's exp do not.  x = k ln2 + r with k the nearest
// integer to x / ln2 (the 1.5 * 2^52 shift) and ln2 split Cody-Waite style (k * hi is exact), |r| <= ln2 / 2; exp(r)
// is its Taylor series to r^13 (truncation below 2^-57), evaluated as 1 + (r + r^2 q(r)).  Results in [-745, 0]
// are within one ulp of the exact value (DESIGN.md §3, "Policy steps").  A subnormal result is scaled in two steps,
// the last one a multiplication, so it is rounded once as IEEE rounds it.  x <= -746 (and -inf) gives 0.
BSB_HD double bsb_exp(double x) {
  if (!(x > -746.0)) return x != x ? x : 0.0;
  if (x > 709.8) return INFINITY;
  const double shift = 6755399441055744.0;
  const double kd = (x * 1.4426950408889634 + shift) - shift;
  const double r = (x - kd * 0.6931471803691238) - kd * 1.9082149292705877e-10;
  double q = 1.6059043836821613e-10;
  q = q * r + 2.08767569878681e-09;
  q = q * r + 2.505210838544172e-08;
  q = q * r + 2.755731922398589e-07;
  q = q * r + 2.7557319223985893e-06;
  q = q * r + 2.48015873015873e-05;
  q = q * r + 0.0001984126984126984;
  q = q * r + 0.001388888888888889;
  q = q * r + 0.008333333333333333;
  q = q * r + 0.041666666666666664;
  q = q * r + 0.16666666666666666;
  q = q * r + 0.5;
  const double p = 1.0 + (r + (r * r) * q);
  const int k = (int)kd;
  if (k < -1021) return ldexp(p, k + 600) * 2.409919865102884e-181;      // 2^-600
  return ldexp(p, k);
}

// Agents' action selection inside a budgeted step (bsb_step_budgeted_policy).  Lane g's draw at global step s is the
// Philox block at counter (s, 0, 0, STREAM_POLICY) with key (seed, g); w0 decides exploration, lo32(w1) picks among
// actions (multiply-shift, as ActionStream maps a chunk) and w1 >> 11 places softmax's target.
enum : int32_t { POLICY_EPSILON_GREEDY = 0, POLICY_SOFTMAX = 1 };

// The action `kind` picks from `row` (n floats: action values or logits).  A row with NaN, or for softmax a row with
// +inf or without a finite entry, sets `invalid` and gets a uniform pick.  Epsilon-greedy: with u = (w0 >> 11) 2^-53,
// u < epsilon explores uniformly; otherwise the pick is among the k entries equal to the row's maximum (±inf are
// ordinary values), in ascending order.  Softmax: weights bsb_exp(l_a - max) (-inf weighs 0), the first action whose
// running sum exceeds u' * sum with u' = (w1 >> 11) 2^-53, or the last action of positive weight when rounding leaves
// none.  The weights are computed twice rather than stored, since a row may be of any length.
BSB_HD int32_t select_action(int32_t kind, const float* row, int32_t n, double epsilon, u64 seed, u64 global_lane,
                             u64 step, bool& invalid) {
  const PhiloxBlock b = philox4x64_10(step, 0, 0, STREAM_POLICY, seed, global_lane);
  const u32 pick = (u32)b.v1;
  float m = -INFINITY;
  bool nan = false;
  for (int32_t a = 0; a < n; ++a) {
    const float v = row[a];
    if (v != v) nan = true;
    else if (v > m) m = v;
  }
  const int32_t uniform = (int32_t)(((u64)pick * (u64)(u32)n) >> 32);
  if (nan || (kind == POLICY_SOFTMAX && (m == INFINITY || m == -INFINITY))) { invalid = true; return uniform; }
  if (kind == POLICY_EPSILON_GREEDY) {
    if ((double)(b.v0 >> 11) * 1.1102230246251565e-16 < epsilon) return uniform;      // 2^-53
    u32 k = 0;
    for (int32_t a = 0; a < n; ++a) k += row[a] == m ? 1u : 0u;
    u32 j = (u32)(((u64)pick * (u64)k) >> 32);
    for (int32_t a = 0; a < n; ++a)
      if (row[a] == m && j-- == 0u) return a;
    return n - 1;
  }
  const double top = (double)m;
  double total = 0.0;
  for (int32_t a = 0; a < n; ++a) total += bsb_exp((double)row[a] - top);
  const double target = ((double)(b.v1 >> 11) * 1.1102230246251565e-16) * total;
  double run = 0.0;
  int32_t last = 0;
  for (int32_t a = 0; a < n; ++a) {
    const double w = bsb_exp((double)row[a] - top);
    run += w;
    if (w > 0.0) last = a;
    if (run > target) return a;
  }
  return last;
}

// Replay sampling (bsb_replay_sample): sample j of global lane g at call index s and draw d is word j & 3 of the Philox
// block at counter (s, d, j >> 2, STREAM_REPLAY) with key (seed, g), mapped onto the n filled slots by multiply-shift
// of its low 32 bits (n <= 2^31 - 1).  Stateless, like the policy stream.
BSB_HD u64 replay_word(const PhiloxBlock& b, int64_t j) {
  switch (j & 3) { case 0: return b.v0; case 1: return b.v1; case 2: return b.v2; default: return b.v3; }
}
BSB_HD int64_t replay_slot(u64 word, int64_t n) { return (int64_t)(((word & 0xffffffffull) * (u64)n) >> 32); }

// log(x) for x in (0, 1] built from + - * / and frexp / ldexp alone, so the host path and the kernels (compiled with
// --fmad=false / -ffp-contract=off) compute the same bits, as bsb_exp does.  x = m 2^k with m in [sqrt(1/2), sqrt(2));
// with f = m - 1 (exact) and s = f / (2 + f), log(m) = f - f^2/2 + s (f^2/2 + R(s^2)), R the minimax series of
// 2 atanh(s) / s - 2 - 2 s^2 / 3 ... in s^2 to degree 7 (FreeBSD's msun e_log.c coefficients); k ln2 is added in
// Cody-Waite halves as bsb_exp splits it.  Within one ulp of numpy.log on (0, 1] (DESIGN.md §3, "Ensemble steps and
// bootstrap samples").  0 gives -inf, anything else outside (0, 1] NaN.
BSB_HD double bsb_log(double x) {
  if (!(x > 0.0 && x <= 1.0)) return x == 0.0 ? -INFINITY : NAN;
  int k;
  double m = frexp(x, &k);               // m in [1/2, 1)
  if (m < 0.7071067811865476) { m = m + m; k -= 1; }
  const double f = m - 1.0;
  const double s = f / (2.0 + f);
  const double z = s * s, w = z * z;
  const double t1 = w * (3.999999999940941908e-01 + w * (2.222219843214978396e-01 + w * 1.531383769920937332e-01));
  const double t2 = z * (6.666666666666735130e-01 + w * (2.857142874366239149e-01 + w * (1.818357216161805012e-01 +
                                                                                         w * 1.479819860511658591e-01)));
  const double R = t2 + t1;
  const double hfsq = 0.5 * f * f;
  const double dk = (double)k;
  return dk * 6.93147180369123816490e-01 - ((hfsq - (s * (hfsq + R) + dk * 1.90821492927058770002e-10)) - f);
}

// Boot_dqn's per-episode head (bsb_step_budgeted_ensemble): a lane whose step ended an episode at global step s draws
// head (lo32(w0) * K) >> 32, w0 word 0 of the Philox block at counter (s, 0, 0, STREAM_HEAD) with key (seed, g).
BSB_HD int32_t ensemble_head(u64 seed, u64 global_lane, u64 step, int32_t num_heads) {
  const PhiloxBlock b = philox4x64_10(step, 0, 0, STREAM_HEAD, seed, global_lane);
  return (int32_t)(((b.v0 & 0xffffffffull) * (u64)(u32)num_heads) >> 32);
}

// Boot_dqn's bootstrap mask and reward noise of transition j (the lane's 0-based count of transitions added before
// it) of global lane g, head k, key (seed, g) (bsb_replay_sample_bootstrap).  Mask: word k & 3 of the block at counter
// (j, k >> 2, 0, STREAM_BOOTSTRAP) gives u = (w >> 11) 2^-53, and the mask is u < mask_prob.  Noise: numpy's legacy
// polar method on the blocks at counter (j, k, 1 + a, STREAM_BOOTSTRAP), attempt a = 0, 1, ...: x, y = 2 u - 1 from
// words 0 and 1, accepted when 0 < r2 = x^2 + y^2 < 1, z = y sqrt(-2 bsb_log(r2) / r2) (gauss's first variate); 0
// after 64 rejected attempts (probability below 1e-42).
BSB_HD uint8_t bootstrap_mask_word(u64 w, double mask_prob) {
  return (double)(w >> 11) * 1.1102230246251565e-16 < mask_prob ? 1 : 0;      // 2^-53
}
BSB_HD PhiloxBlock bootstrap_mask_block(u64 seed, u64 global_lane, u64 j, u64 k4) {
  return philox4x64_10(j, k4, 0, STREAM_BOOTSTRAP, seed, global_lane);
}
BSB_HD float bootstrap_noise(u64 seed, u64 global_lane, u64 j, u64 k) {
  for (u64 attempt = 0; attempt < 64; ++attempt) {
    const PhiloxBlock b = philox4x64_10(j, k, 1 + attempt, STREAM_BOOTSTRAP, seed, global_lane);
    const double x = 2.0 * ((double)(b.v0 >> 11) * 1.1102230246251565e-16) - 1.0;
    const double y = 2.0 * ((double)(b.v1 >> 11) * 1.1102230246251565e-16) - 1.0;
    const double r2 = x * x + y * y;
    if (r2 < 1.0 && r2 != 0.0) return (float)(y * sqrt(-2.0 * bsb_log(r2) / r2));
  }
  return 0.0f;
}

// ---------------------------------------------------------------------------
// Bit source 1: Philox stream with numpy's buffering semantics.
//   numpy keeps a 4-word buffer; the counter is incremented BEFORE a block is
//   generated, so word w of the stream is word (w & 3) of the block at counter
//   (w >> 2) + 1.  next_uint32 returns the low half of a fresh 64-bit word and
//   keeps the high half for the next call.
// Persistent state per lane is ONE u64:
//   bits  0..53  words consumed so far
//   bits 54..61  d: a saved high half is pending from word (pos - d); 0 = none.
//                (next_uint64 calls do not disturb numpy's saved half, so it can
//                lag behind pos: by at most num_bits + 1 <= 65 words here.)
//   bit  62      a cached gaussian is pending (value kept in a separate array)
// ---------------------------------------------------------------------------
static const u64 RNG_HASGAUSS = 1ull << 62;
static const u64 RNG_POSMASK = (1ull << 54) - 1;
static const int RNG_LAG_SHIFT = 54;
static const u64 RNG_LAG_MAX = 255;

struct PhiloxSrc {
  u64 k0, k1, stream;
  u64 pos;          // 64-bit words consumed
  u64 pend;         // 1 + index of the word whose high half is saved (0 = none)
  u64 blk;          // counter value of the buffered block (0 = none)
  u64 b0, b1, b2, b3;

  BSB_HD void open(u64 seed, u64 global_lane, u64 stream_id, u64 packed) {
    k0 = seed; k1 = global_lane; stream = stream_id;
    pos = packed & RNG_POSMASK;
    const u64 lag = (packed >> RNG_LAG_SHIFT) & RNG_LAG_MAX;
    pend = lag ? (pos - lag + 1) : 0;
    blk = 0; b0 = b1 = b2 = b3 = 0;
  }
  BSB_HD u64 packed() const {
    u64 lag = pend ? (pos - (pend - 1)) : 0;
    if (lag > RNG_LAG_MAX) lag = 0;   // unreachable for the supported families (see header)
    return pos | (lag << RNG_LAG_SHIFT);
  }
  static BSB_HD u64 pick(const PhiloxBlock& b, u32 i) { return i == 0 ? b.v0 : (i == 1 ? b.v1 : (i == 2 ? b.v2 : b.v3)); }

  BSB_HD u64 next64() {
    const u64 want = (pos >> 2) + 1;
    if (want != blk) {
      const PhiloxBlock b = philox4x64_10(want, 0, 0, stream, k0, k1);
      b0 = b.v0; b1 = b.v1; b2 = b.v2; b3 = b.v3; blk = want;
    }
    const u32 i = (u32)(pos & 3);
    ++pos;
    return i == 0 ? b0 : (i == 1 ? b1 : (i == 2 ? b2 : b3));
  }
  BSB_HD u32 next32() {
    if (pend) {
      const u64 w = pend - 1;
      pend = 0;
      const u64 want = (w >> 2) + 1;
      if (want == blk) { const u32 i = (u32)(w & 3); return (u32)((i == 0 ? b0 : (i == 1 ? b1 : (i == 2 ? b2 : b3))) >> 32); }
      return (u32)(pick(philox4x64_10(want, 0, 0, stream, k0, k1), (u32)(w & 3)) >> 32);
    }
    const u64 v = next64();
    pend = pos;   // word index pos - 1, stored + 1
    return (u32)v;
  }
  BSB_HD double next_double() { return (double)(next64() >> 11) * (1.0 / 9007199254740992.0); }
  // next_double() > 0.5 without floating point: (w >> 11) * 2^-53 > 1/2  <=>  (w >> 11) > 2^52  <=>  w >= 2^63 + 2^11
  BSB_HD bool next_above_half() { return next64() >= 0x8000000000000800ull; }

  // The next `n` (<= 64) Bernoulli(1/2) draws as bits of the result (draw k -> bit k): binomial(1, .5, size=n).
  // Once the position is block-aligned, TWO Philox blocks (8 draws) are computed per iteration; the ten-round
  // chains are independent, so the scheduler interleaves them and the integer-multiply latency that bounds a
  // single chain is overlapped (umbrella_chain draws up to 100 of these per lane-step, memory_chain 40 per reset).
  // Four chains at once would cost registers.
  static BSB_HD u64 nibble(const PhiloxBlock& b, u64 T) {
    return (u64)(b.v0 >= T) | ((u64)(b.v1 >= T) << 1) | ((u64)(b.v2 >= T) << 2) | ((u64)(b.v3 >= T) << 3);
  }
  BSB_HD u64 next_half_bits(int n) {
    const u64 T = 0x8000000000000800ull;
    u64 bits = 0;
    int k = 0;
    while (k < n && (pos & 3) != 0) { bits |= (u64)next_above_half() << k; ++k; }
    while (n - k >= 8) {
      const u64 c = (pos >> 2) + 1;
      const PhiloxBlock x = philox4x64_10(c, 0, 0, stream, k0, k1);
      const PhiloxBlock y = philox4x64_10(c + 1, 0, 0, stream, k0, k1);
      bits |= (nibble(x, T) | (nibble(y, T) << 4)) << k;
      k += 8; pos += 8;
    }
    while (k < n) { bits |= (u64)next_above_half() << k; ++k; }
    return bits;
  }
};

// ---------------------------------------------------------------------------
// Bit source 2: MT19937 with numpy's legacy integer seeding.  The 624-word key
// lives in caller memory with element stride `stride` (device: [624][B]
// lane-minor so that lanes at the same index coalesce; host: stride 1).
// ---------------------------------------------------------------------------
struct MtSrc {
  u32* key; int64_t stride; int32_t idx;

  BSB_HD void open(u32* key_, int64_t stride_, int32_t idx_) { key = key_; stride = stride_; idx = idx_; }
  BSB_HD u32& at(int i) { return key[(int64_t)i * stride]; }

  static BSB_HD u32 twist(u32 cur, u32 nxt, u32 far) {
    const u32 y = (cur & 0x80000000u) | (nxt & 0x7fffffffu);
    return far ^ (y >> 1) ^ ((y & 1u) ? 0x9908b0dfu : 0u);
  }
  BSB_HD void regenerate() {
    for (int k = 0; k < 624 - 397; ++k) at(k) = twist(at(k), at(k + 1), at(k + 397));
    for (int k = 624 - 397; k < 623; ++k) at(k) = twist(at(k), at(k + 1), at(k - (624 - 397)));
    at(623) = twist(at(623), at(0), at(396));
    idx = 0;
  }
  BSB_HD u32 next32() {
    if (idx >= 624) regenerate();
    u32 y = at(idx++);
    y ^= (y >> 11);
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= (y >> 18);
    return y;
  }
  BSB_HD double next_double() {
    const u32 a = next32() >> 5, b = next32() >> 6;
    return ((double)a * 67108864.0 + (double)b) / 9007199254740992.0;
  }
  // next_double() > 0.5: the numerator a * 2^26 + b is an exact 53-bit integer; compare it with 2^52
  BSB_HD bool next_above_half() {
    const u32 a = next32() >> 5, b = next32() >> 6;
    return (((u64)a << 26) | (u64)b) > (1ull << 52);
  }
  BSB_HD u64 next_half_bits(int n) {
    u64 bits = 0;
    for (int k = 0; k < n; ++k) bits |= (u64)next_above_half() << k;
    return bits;
  }
};

// numpy's legacy seeding of MT19937 from one 32-bit integer.
inline void mt19937_seed_host(u32* key, int64_t stride, u32 seed) {
  for (int i = 0; i < 624; ++i) {
    key[(int64_t)i * stride] = seed;
    seed = 1812433253u * (seed ^ (seed >> 30)) + (u32)i + 1u;
  }
}

// ---------------------------------------------------------------------------
// numpy legacy distributions over either bit source.  `Gauss` is the cached
// second variate of the polar method (RandomState's has_gauss / gauss).
// ---------------------------------------------------------------------------
struct GaussCache { int has; double value; };

template <class Src>
struct LegacyRng {
  Src src;
  GaussCache g;

  BSB_HD double rand() { return src.next_double(); }

  BSB_HD double uniform(double low, double high) {
    const double range = high - low;
    return low + range * src.next_double();
  }
  // binomial(n=1, p=0.5): inversion with qn = exp(log(0.5)) = 0.5, bound = 1.
  BSB_HD int binomial_half() { return src.next_above_half() ? 1 : 0; }
  // binomial(1, 0.5, size=n), n <= 64, draw k in bit k
  BSB_HD u64 binomial_half_bits(int n) { return src.next_half_bits(n); }

  // randint(n) for 1 <= n <= 2^32.
  BSB_HD u32 randint(u32 n) {
    const u32 rng = n - 1u;
    if (rng == 0u) return 0u;
    u32 mask = rng;
    mask |= mask >> 1; mask |= mask >> 2; mask |= mask >> 4; mask |= mask >> 8; mask |= mask >> 16;
    u32 v;
    do { v = src.next32() & mask; } while (v > rng);
    return v;
  }
  BSB_HD double randn() {
    if (g.has) { g.has = 0; const double t = g.value; g.value = 0.0; return t; }
    double x1, x2, r2;
    do {
      x1 = 2.0 * src.next_double() - 1.0;
      x2 = 2.0 * src.next_double() - 1.0;
      r2 = x1 * x1 + x2 * x2;
    } while (r2 >= 1.0 || r2 == 0.0);
    const double f = sqrt(-2.0 * log(r2) / r2);
    g.value = f * x1; g.has = 1;
    return f * x2;
  }
};

}  // namespace bsb
