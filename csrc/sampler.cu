// Fused sampler for sm_90a: repetition penalty (seen-token bitmap) -> temperature ->
// exact top-p via two-level radix histogram of the probability bits -> multinomial draw
// (or argmax when temperature <= 0).  One CTA per sequence, logits are fp32 [B, ld] as
// written by the lm_head GEMM.  The sampled id is stored locally (token ring, history
// bitmap) and, on the last piece of a pipeline, straight into piece 0's token buffer on
// the peer GPU followed by a release flag (4 bytes/sequence over NVLink, no NCCL).
//
// Semantics follow the reference's generation defaults (bee2bee/hf.py:91-105):
// repetition_penalty 1.15, top_p 0.95, do_sample iff temperature > 0, greedy otherwise.
//
// Performance notes: every pass over the 128k logits is
// L2-latency bound, so logits are read 8 at a time per thread (2 x 128-bit loads in flight);
// histogram mass is accumulated in 32.32 fixed point with native 32-bit shared-memory atomics
// (float / 64-bit shared atomics are CAS loops).
#include "kernels.h"

#include "common.cuh"
#include "launch.cuh"

namespace b2b {

constexpr int SAMP_THREADS = 1024;
constexpr int NBINS = 4096;

__device__ __forceinline__ uint32_t hash_u32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  return x;
}

struct SampleParams {
  const float* logits;      // [B, ld]
  uint32_t* seen;           // [rows, ceil(V/32)] bitmap of ids in the context, or null
  int* out_tokens;          // [rows] local
  int* peer_tokens;         // [rows] on piece 0 (may be == out_tokens / null)
  int* history;             // [rows, hist_stride] token ring, or null
  const int* hist_pos;      // [rows] write index into history
  int* hist_pos_out;        // [rows] incremented copy
  int hist_stride;
  int vocab;
  int ld;                   // row stride of logits (vocab padded to a GEMM tile)
  float softcap;            // final-logit soft-capping (Gemma-2), 0 = off
  const float* temperature; // [rows]
  const float* top_p;       // [rows]
  const float* rep_penalty; // [rows]
  const uint32_t* seeds;    // [rows]
  const uint32_t* step;     // device step counter (rng stream), may be null
  uint32_t* signal_flag;    // peer flag (token handoff) or null
  uint32_t* signal_epoch;   // local epoch for the flag
  uint32_t* done_counter;   // local, self-resetting
  const int* row_map;       // optional [batch]: per-sequence state of logits row b lives at row row_map[b]; < 0 = skip the row
};

// logit -> (soft-cap) -> repetition penalty -> temperature
__device__ __forceinline__ float transform(float l, bool is_seen, float pen, float inv_temp, float cap) {
  if (cap > 0.f) l = cap * tanhf(l / cap);
  if (is_seen) l = l > 0.f ? l / pen : l * pen;
  return l * inv_temp;
}

constexpr int SBINS = 2048;          // histogram bins per level (11 + 11 bits of the 28-bit key)
constexpr int MAX_CS = 8;            // portable cluster size
constexpr int MAX_SLICE = 36864;     // ids per CTA kept in shared memory (144 KB)

// Control block at the start of dynamic shared memory; the CTA's slice of exp'd logits follows it.
struct __align__(16) SampShared {
  uint32_t h1_lo[SBINS], h1_hi[SBINS];      // level-1 histogram, 32.32 fixed point split in two native-atomic words
  uint32_t h2_lo[SBINS], h2_hi[SBINS];      // level-2 histogram (inside the boundary bin)
  unsigned long long merged[SBINS];         // cluster-wide sum of the level being scanned
  unsigned long long wsum[32];
  unsigned long long red_u[32];
  unsigned long long cz[MAX_CS];            // per-CTA partition-function partials (written by every peer)
  float cmax[MAX_CS];
  int camx[MAX_CS];
  float ctot[MAX_CS];                       // per-CTA kept mass
  float red_f[32];
  int red_i[32];
  float wtot[32];
  unsigned long long s_u[2];
  int s_i[4];
};

__device__ __forceinline__ void cluster_sync_all() {
  cluster_arrive_release();
  cluster_wait_acquire();
}

// monotone 28-bit key of e in [2^-32, 1]: 5 exponent bits + 23 mantissa bits (smaller e -> 0)
__device__ __forceinline__ uint32_t dkey(float e) {
  const uint32_t u = __float_as_uint(e);
  return u < 0x2F800000u ? 0u : min(u - 0x2F800000u, 0x0FFFFFFFu);
}
__device__ __forceinline__ uint32_t fx32(float e) { return static_cast<uint32_t>(fminf(e * 4294967296.0f, 4294967040.0f)); }
__device__ __forceinline__ void hist_add(uint32_t* lo, uint32_t* hi, int bin, uint32_t f) {
  const uint32_t old = atomicAdd(&lo[bin], f);
  if (old + f < old) atomicAdd(&hi[bin], 1u);
}

// One CLUSTER of CS CTAs per sequence (grid = [B, 1, CS]); CTA r owns ids [r*W, (r+1)*W).  A single
// SM is instruction-bound on a 128k vocabulary, so the
// vocabulary is spread over CS SMs, each slice is read from L2 exactly once and then lives in shared
// memory as exp(l - max); the per-level histograms are merged across the cluster through DSMEM.
__global__ void __launch_bounds__(SAMP_THREADS, 1) sample_kernel(const SampleParams p, const int W) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  SampShared& S = *reinterpret_cast<SampShared*>(smem_raw);
  float* ebuf = reinterpret_cast<float*>(smem_raw + sizeof(SampShared));

  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int CS = gridDim.z, r = blockIdx.z;
  // Distributed shared memory of a peer may only be touched once that CTA has started executing: every thread
  // arrives on the cluster barrier here and waits on it right before the first remote store (compute-sanitizer:
  // "block that might not have entered yet").
  cluster_arrive_release();
  pdl_launch_dependents();
  for (int i = tid; i < SBINS; i += SAMP_THREADS) { S.h1_lo[i] = 0u; S.h1_hi[i] = 0u; S.h2_lo[i] = 0u; S.h2_hi[i] = 0u; }
  pdl_wait();

  const int bb = (p.row_map != nullptr) ? p.row_map[b] : b;           // row of the per-sequence state
  // the flag handoff counts one arrival per sequence (cluster), sampled or skipped
  auto arrive = [&]() {
    if (p.signal_flag != nullptr) {
      __threadfence_system();
      const uint32_t prev = atomicAdd(p.done_counter, 1u);
      if (prev == gridDim.x - 1) {
        __threadfence_system();
        *p.done_counter = 0;
        const uint32_t e = *reinterpret_cast<volatile uint32_t*>(p.signal_epoch) + 1;
        *reinterpret_cast<volatile uint32_t*>(p.signal_epoch) = e;
        st_release_sys(p.signal_flag, e);
      }
    }
  };
  if (bb < 0) {
    // padded / not-yet-complete row of a prefill chunk (cluster-uniform decision): nothing to sample
    cluster_wait_acquire();
    if (r == 0 && tid == 0) arrive();
    return;
  }
  const int V = p.vocab;
  const float* logits = p.logits + static_cast<size_t>(b) * p.ld;
  const bool vec_ok = (reinterpret_cast<uintptr_t>(logits) & 15) == 0;
  const float cap = p.softcap;
  uint32_t* seen = p.seen ? p.seen + static_cast<size_t>(bb) * ((V + 31) / 32) : nullptr;
  const float temp = p.temperature ? p.temperature[bb] : 0.f;
  const float pen = p.rep_penalty ? p.rep_penalty[bb] : 1.f;
  const float top_p = p.top_p ? fminf(p.top_p[bb], 1.f) : 1.f;
  const bool greedy = !(temp > 0.f);
  const float inv_temp = greedy ? 1.f : 1.f / temp;
  const uint32_t* seen_r = (pen != 1.f) ? seen : nullptr;
  const int lo = min(V, r * W), hi = min(V, lo + W), n = hi - lo;
  const int n4 = n >> 2;

  // exactly one thread per sequence publishes the token
  auto publish = [&](int token) {
    p.out_tokens[bb] = token;
    if (seen != nullptr) atomicOr(&seen[token >> 5], 1u << (token & 31));
    if (p.history != nullptr) {
      const int pos = p.hist_pos[bb];
      // the history is a ring: the host reads each burst's window before the writer can lap it
      p.history[static_cast<size_t>(bb) * p.hist_stride + (pos % p.hist_stride)] = token;
      p.hist_pos_out[bb] = pos + 1;
    }
    if (p.peer_tokens != nullptr && p.peer_tokens != p.out_tokens) p.peer_tokens[bb] = token;
    arrive();
  };

  // ---- phase 1: L2 -> (soft-cap, penalty, temperature) -> shared memory; running max / argmax
  float mx = -INFINITY; int amx = 0;
  {
    auto take = [&](int i, float raw, uint32_t sw) {
      const float l = transform(raw, (sw >> (i & 31)) & 1u, pen, inv_temp, cap);
      ebuf[i - lo] = l;
      if (l > mx) { mx = l; amx = i; }
    };
    for (int q = tid; q < n4; q += 2 * SAMP_THREADS) {
      const int q2 = q + SAMP_THREADS;
      const bool has2 = q2 < n4;
      const int i0 = lo + 4 * q, i1 = lo + 4 * q2;
      float a[4], c[4] = {0.f, 0.f, 0.f, 0.f};
      if (vec_ok) {
        const float4 va = *reinterpret_cast<const float4*>(logits + i0);
        a[0] = va.x; a[1] = va.y; a[2] = va.z; a[3] = va.w;
        if (has2) {
          const float4 vc = *reinterpret_cast<const float4*>(logits + i1);
          c[0] = vc.x; c[1] = vc.y; c[2] = vc.z; c[3] = vc.w;
        }
      } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) a[k] = logits[i0 + k];
        if (has2) {
#pragma unroll
          for (int k = 0; k < 4; ++k) c[k] = logits[i1 + k];
        }
      }
      const uint32_t sa = seen_r ? seen_r[i0 >> 5] : 0u;
      const uint32_t sc = (seen_r && has2) ? seen_r[i1 >> 5] : 0u;
#pragma unroll
      for (int k = 0; k < 4; ++k) take(i0 + k, a[k], sa);
      if (has2) {
#pragma unroll
        for (int k = 0; k < 4; ++k) take(i1 + k, c[k], sc);
      }
    }
    for (int i = lo + 4 * n4 + tid; i < hi; i += SAMP_THREADS) take(i, logits[i], seen_r ? seen_r[i >> 5] : 0u);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, mx, o);
    const int oi = __shfl_xor_sync(0xffffffffu, amx, o);
    if (om > mx || (om == mx && oi < amx)) { mx = om; amx = oi; }
  }
  if (lane == 0) { S.red_f[warp] = mx; S.red_i[warp] = amx; }
  __syncthreads();
  cluster_wait_acquire();            // all CTAs of the cluster are running (pairs with the arrive at kernel entry)
  if (warp == 0) {
    mx = S.red_f[lane]; amx = S.red_i[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float om = __shfl_xor_sync(0xffffffffu, mx, o);
      const int oi = __shfl_xor_sync(0xffffffffu, amx, o);
      if (om > mx || (om == mx && oi < amx)) { mx = om; amx = oi; }
    }
    if (lane < CS) {       // every peer (and this CTA) gets this CTA's partial
      st_dsmem_f32(mapa_smem(smem_u32(&S.cmax[r]), lane), mx);
      st_dsmem_u32(mapa_smem(smem_u32(&S.camx[r]), lane), static_cast<uint32_t>(amx));
    }
  }
  cluster_sync_all();
  mx = S.cmax[0];
  int token = S.camx[0];
  for (int c = 1; c < CS; ++c)
    if (S.cmax[c] > mx) { mx = S.cmax[c]; token = S.camx[c]; }      // ties keep the lower rank = lower id

  if (greedy) {
    if (r == 0 && tid == 0) publish(token);
    return;
  }

  // ---- phase 2: e = exp(l - max) in place; level-1 histogram (top 11 key bits) and partition function
  unsigned long long zsum = 0ull;
  {
    float4* e4 = reinterpret_cast<float4*>(ebuf);
    for (int q = tid; q < n4; q += SAMP_THREADS) {
      float4 v = e4[q];
      v.x = __expf(v.x - mx); v.y = __expf(v.y - mx); v.z = __expf(v.z - mx); v.w = __expf(v.w - mx);
      e4[q] = v;
      const float ev[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t f = fx32(ev[k]);
        zsum += f;
        hist_add(S.h1_lo, S.h1_hi, dkey(ev[k]) >> 17, f);
      }
    }
    for (int j = 4 * n4 + tid; j < n; j += SAMP_THREADS) {
      const float e = __expf(ebuf[j] - mx);
      ebuf[j] = e;
      const uint32_t f = fx32(e);
      zsum += f;
      hist_add(S.h1_lo, S.h1_hi, dkey(e) >> 17, f);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) zsum += __shfl_xor_sync(0xffffffffu, zsum, o);
  if (lane == 0) S.red_u[warp] = zsum;
  __syncthreads();
  if (warp == 0) {
    unsigned long long z = S.red_u[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
    if (lane < CS) st_dsmem_u64(mapa_smem(smem_u32(&S.cz[r]), lane), z);
  }
  cluster_sync_all();

  // cluster-wide histogram -> S.merged (every CTA computes the same sum), then a top-down search for the
  // highest bin whose suffix mass (plus `carry`) reaches `need`.  Results: s_i[0] = bin, s_u[0] = mass above it.
  auto merge_and_find = [&](uint32_t* hlo, uint32_t* hhi, unsigned long long carry, unsigned long long need) {
    {
      const int bin = 2 * tid;        // SBINS == 2 * SAMP_THREADS
      unsigned long long m0 = 0ull, m1 = 0ull;
      const uint32_t alo = smem_u32(&hlo[bin]), ahi = smem_u32(&hhi[bin]);
      for (int c = 0; c < CS; ++c) {
        const uint2 l2 = ld_dsmem_v2u32(mapa_smem(alo, c));
        const uint2 h2 = ld_dsmem_v2u32(mapa_smem(ahi, c));
        m0 += (static_cast<unsigned long long>(h2.x) << 32) | l2.x;
        m1 += (static_cast<unsigned long long>(h2.y) << 32) | l2.y;
      }
      S.merged[bin] = m0; S.merged[bin + 1] = m1;
      unsigned long long ws = m0 + m1;      // warp w covers bins [64w, 64w + 64)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) ws += __shfl_xor_sync(0xffffffffu, ws, o);
      if (lane == 0) S.wsum[warp] = ws;
    }
    __syncthreads();
    if (warp == 0) {
      // lane l looks at warp-chunk 31 - l (highest bins first)
      const unsigned long long v = S.wsum[31 - lane];
      unsigned long long pre = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const unsigned long long t = __shfl_up_sync(0xffffffffu, pre, o); if (lane >= o) pre += t; }
      const unsigned ball = __ballot_sync(0xffffffffu, carry + pre >= need);
      int found = -1;
      unsigned long long above = carry;
      if (ball) {
        const int l0 = __ffs(ball) - 1;
        unsigned long long run = carry + __shfl_sync(0xffffffffu, pre, l0) - __shfl_sync(0xffffffffu, v, l0);
        const int cbase = (31 - l0) * 64;
        for (int base = cbase + 32; base >= cbase && found < 0; base -= 32) {
          const unsigned long long bv = S.merged[base + (31 - lane)];
          unsigned long long bp = bv;
#pragma unroll
          for (int o = 1; o < 32; o <<= 1) { const unsigned long long t = __shfl_up_sync(0xffffffffu, bp, o); if (lane >= o) bp += t; }
          const unsigned hit = __ballot_sync(0xffffffffu, run + bp >= need);
          if (hit) {
            const int l1 = __ffs(hit) - 1;
            found = base + (31 - l1);
            above = run + __shfl_sync(0xffffffffu, bp, l1) - __shfl_sync(0xffffffffu, bv, l1);
          } else {
            run += __shfl_sync(0xffffffffu, bp, 31);
          }
        }
      }
      if (lane == 0) { S.s_i[0] = found < 0 ? 0 : found; S.s_u[0] = found < 0 ? carry : above; }
    }
    __syncthreads();
  };

  unsigned long long Z = 0ull;
  for (int c = 0; c < CS; ++c) Z += S.cz[c];
  const unsigned long long need = static_cast<unsigned long long>(static_cast<double>(top_p) * static_cast<double>(Z));
  merge_and_find(S.h1_lo, S.h1_hi, 0ull, need);
  const int B1 = S.s_i[0];
  const unsigned long long above1 = S.s_u[0];       // mass strictly above the boundary bin
  __syncthreads();                                   // s_i / merged are reused by the second level

  // ---- phase 3: level-2 histogram inside the boundary bin (next 11 key bits)
  {
    const float4* e4 = reinterpret_cast<const float4*>(ebuf);
    for (int q = tid; q < n4; q += SAMP_THREADS) {
      const float4 v = e4[q];
      const float ev[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint32_t d = dkey(ev[k]);
        if (static_cast<int>(d >> 17) == B1) hist_add(S.h2_lo, S.h2_hi, (d >> 6) & (SBINS - 1), fx32(ev[k]));
      }
    }
    for (int j = 4 * n4 + tid; j < n; j += SAMP_THREADS) {
      const uint32_t d = dkey(ebuf[j]);
      if (static_cast<int>(d >> 17) == B1) hist_add(S.h2_lo, S.h2_hi, (d >> 6) & (SBINS - 1), fx32(ebuf[j]));
    }
  }
  __syncthreads();
  cluster_sync_all();
  merge_and_find(S.h2_lo, S.h2_hi, above1, need);
  const uint32_t thr = (static_cast<uint32_t>(B1) << 17) | (static_cast<uint32_t>(S.s_i[0]) << 6);

  // ---- phase 4: multinomial draw over the kept set {dkey(e) >= thr}, in id order.
  // warp w owns a contiguous chunk of this CTA's slice; lanes own interleaved quads.
  const int cw = ((n + 31) / 32 + 127) & ~127;
  const int c0 = min(n, warp * cw), c1 = min(n, c0 + cw);
  float mine = 0.f;
  {
    const float4* e4 = reinterpret_cast<const float4*>(ebuf + c0);
    const int nq = (c1 - c0) >> 2;
    for (int q = lane; q < nq; q += 32) {
      const float4 v = e4[q];
      if (dkey(v.x) >= thr) mine += v.x;
      if (dkey(v.y) >= thr) mine += v.y;
      if (dkey(v.z) >= thr) mine += v.z;
      if (dkey(v.w) >= thr) mine += v.w;
    }
    for (int j = c0 + 4 * nq + lane; j < c1; j += 32)
      if (dkey(ebuf[j]) >= thr) mine += ebuf[j];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
  if (lane == 0) S.wtot[warp] = mine;
  __syncthreads();
  // inclusive prefix over the 32 warp totals (every warp computes the same values)
  const float wt = S.wtot[lane];
  float wpre = wt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const float t = __shfl_up_sync(0xffffffffu, wpre, o); if (lane >= o) wpre += t; }
  const float cta_total = __shfl_sync(0xffffffffu, wpre, 31);
  if (warp == 0 && lane < CS) st_dsmem_f32(mapa_smem(smem_u32(&S.ctot[r]), lane), cta_total);
  cluster_sync_all();                 // last remote access of the kernel (also fences the DSMEM histogram reads)

  float kept_total = 0.f, my_excl = 0.f;
  for (int c = 0; c < CS; ++c) { if (c == r) my_excl = kept_total; kept_total += S.ctot[c]; }
  const uint32_t stepv = p.step ? *p.step : 0u;
  const uint32_t h = hash_u32((p.seeds ? p.seeds[bb] : 0x1234567u) ^ hash_u32(stepv * 0x9E3779B9u + b));
  const float u01 = (static_cast<float>(h >> 8) + 0.5f) * (1.0f / 16777216.0f);
  const float target = u01 * kept_total;
  // the owner is the LAST non-empty CTA whose exclusive prefix is <= target (absorbs float round-off at the far edge)
  int owner = -1;
  {
    float run = 0.f;
    for (int c = 0; c < CS; ++c) {
      if (S.ctot[c] > 0.f && (run <= target || owner < 0)) owner = c;
      run += S.ctot[c];
    }
  }
  if (owner < 0) {                    // only reachable with NaN logits: fall back to the arg-max
    if (r == 0 && tid == 0) publish(token);
    return;
  }
  if (owner != r) return;
  // same rule for the warp inside the CTA
  const float w_excl = my_excl + (wpre - wt);
  const unsigned cand = __ballot_sync(0xffffffffu, wt > 0.f && w_excl <= target);
  const unsigned nonempty = __ballot_sync(0xffffffffu, wt > 0.f);
  const int wsel = cand ? (31 - __clz(cand)) : (__ffs(nonempty) - 1);
  if (warp != wsel) return;
  float run = my_excl + __shfl_sync(0xffffffffu, wpre - wt, wsel);
  int pick = -1, last_kept = -1;
  for (int base = c0; base < c1 && pick < 0; base += 32) {
    const int j = base + lane;
    float v = 0.f;
    if (j < c1) { const float e = ebuf[j]; if (dkey(e) >= thr) v = e; }
    float pre = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const float t = __shfl_up_sync(0xffffffffu, pre, o); if (lane >= o) pre += t; }
    const unsigned kept = __ballot_sync(0xffffffffu, v > 0.f);
    if (kept) last_kept = base + (31 - __clz(kept));
    const unsigned hit = __ballot_sync(0xffffffffu, v > 0.f && run + pre > target);
    if (hit) pick = base + (__ffs(hit) - 1);
    run += __shfl_sync(0xffffffffu, pre, 31);
  }
  if (pick < 0) pick = last_kept;
  if (lane == 0) publish(pick >= 0 ? lo + pick : token);
}

// mark prompt tokens in the seen bitmap: ids [n], seq_of [n]
__global__ void mark_seen_kernel(const int* ids, const int* seq_of, uint32_t* seen, int n, int words, int vocab) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int id = ids[i];
  if (id < 0 || id >= vocab) return;
  atomicOr(&seen[static_cast<size_t>(seq_of[i]) * words + (id >> 5)], 1u << (id & 31));
}

// cluster size: the slice must fit in shared memory; beyond that use more SMs while the grid is below one wave
int sample_cluster_size(int batch, int vocab, int sms) {
  int cs = 1;
  while (cs < MAX_CS && (vocab + cs - 1) / cs > MAX_SLICE) cs *= 2;
  if ((vocab + cs - 1) / cs > MAX_SLICE) return 0;
  while (cs < MAX_CS && batch * cs * 2 <= sms) cs *= 2;
  return cs;
}

int launch_sample(const float* logits, uint32_t* seen, int* out_tokens, int* peer_tokens, int* history,
                  const int* hist_pos, int* hist_pos_out, int hist_stride, int batch, int vocab, int ld, float softcap,
                  const float* temperature, const float* top_p, const float* rep_penalty, const uint32_t* seeds,
                  const uint32_t* step, uint32_t* signal_flag, uint32_t* signal_epoch, uint32_t* done_counter,
                  const int* row_map, cudaStream_t s) {
  SampleParams p;
  p.logits = logits; p.seen = seen; p.out_tokens = out_tokens; p.peer_tokens = peer_tokens; p.history = history;
  p.hist_pos = hist_pos; p.hist_pos_out = hist_pos_out; p.hist_stride = hist_stride; p.vocab = vocab; p.ld = ld; p.softcap = softcap;
  p.temperature = temperature; p.top_p = top_p; p.rep_penalty = rep_penalty; p.seeds = seeds; p.step = step;
  p.signal_flag = signal_flag; p.signal_epoch = signal_epoch; p.done_counter = done_counter; p.row_map = row_map;
  if (sample_cluster_size(1, vocab, 0) == 0) return -6;
  static int sm_count[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  int sms = dev < 64 ? sm_count[dev] : 0;
  if (sms == 0) {
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -9;
    if (dev < 64) sm_count[dev] = sms;
  }
  const int cs = sample_cluster_size(batch, vocab, sms);
  const int W = (((vocab + cs - 1) / cs) + 127) & ~127;
  const size_t smem = sizeof(SampShared) + static_cast<size_t>(W) * sizeof(float);
  static bool attr_set[64] = {};
  if (dev < 64 && !attr_set[dev]) {
    const cudaError_t e = cudaFuncSetAttribute(sample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               static_cast<int>(sizeof(SampShared) + MAX_SLICE * sizeof(float)));
    if (e != cudaSuccess) return static_cast<int>(e);
    attr_set[dev] = true;
  }
  return static_cast<int>(launch_kernel(sample_kernel, dim3(batch, 1, cs), dim3(SAMP_THREADS), smem, s, cs, p, W));
}

int launch_mark_seen(const int* ids, const int* seq_of, uint32_t* seen, int n, int vocab, cudaStream_t s) {
  if (n <= 0) return 0;
  return static_cast<int>(launch_kernel(mark_seen_kernel, dim3((n + 255) / 256), dim3(256), 0, s, 1, ids, seq_of, seen, n,
                                        (vocab + 31) / 32, vocab));
}

}  // namespace b2b
