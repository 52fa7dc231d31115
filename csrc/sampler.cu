// Fused sampler for sm_90a: soft-cap -> logit bias (per-row id / value table) -> repetition penalty (seen-token
// bitmap) -> presence / frequency penalty (per-row counts of generated tokens) -> temperature -> top-k -> top-p ->
// min-p, each decided on a two-level radix histogram of the probability bits ->
// multinomial draw (or argmax when temperature <= 0).  One cluster per sequence, logits are
// fp32 [B, ld] as written by the lm_head GEMM.  The sampled id is stored locally (token ring,
// history bitmap) and, on the last piece of a pipeline, straight into piece 0's token buffer on
// the peer GPU followed by a release flag (4 bytes/sequence over NVLink, no NCCL).
//
// Semantics follow the reference's generation defaults (bee2bee/hf.py:91-105):
// repetition_penalty 1.15, top_p 0.95, do_sample iff temperature > 0, greedy otherwise.
// Logit bias (OpenAI / vLLM `logit_bias`; per row, bias_n = 0 = off) runs right after soft-cap, so the repetition
// penalty's sign test sees the biased logit: l = l + b for each of the row's first min(bias_n, bias_stride) entries;
// other ids are untouched.  The ids of a row must be unique (the host guarantees it); an id outside [0, V) lies in no
// CTA's slice and is ignored.
// Presence / frequency penalties (vLLM / OpenAI; per row, 0 = off) run after the repetition penalty: with c the
// number of times the id has been generated for the row (prompt excluded; an int16 table that saturates at 32767),
// l = (l - f c) - p when c > 0.  With a count table, the publishing thread increments the drawn id's count
// (saturating); every CTA of the cluster has read its counts before the draw.  Greedy rows are biased and penalised
// too.  Both steps round to nearest explicitly (no FMA contraction), so an fp32 reference reproduces them bit for bit.
// After temperature the filters run in transformers' processor order, with e = exp(l - max):
//   * top-k (k per row; k <= 0 or k >= V = off): K = the tokens whose e is at least the k-th
//     largest e, ties at the k-th value kept.  K is decided on the same 22-bit key (top 22 bits
//     of the 28-bit key below) as top-p, so it may also keep tokens whose e lies within one
//     level-2 bin (a relative 2^-18 to 2^-17) below the k-th, and every token with e < 2^-32
//     when the k-th is below 2^-32;
//   * top-p over K: need = min(top_p, 1) Z_K with Z_K the mass of K; the nucleus is the smallest
//     highest-e prefix reaching need (a prefix of K, so it is found on the unchanged mass
//     histograms);
//   * min-p (per row; <= 0 = off): keep e >= min(min_p, 1) on the full 28-bit key, i.e.
//     p >= min_p p_max.
// Every filter keeps a highest-e prefix, so the kept set is {key >= max(thr_k, thr_p, key(min_p))}
// and always holds the maximal tokens.  Greedy rows ignore top-k and min-p.  The branches on
// top-k and min-p are uniform per row: a row with both off runs the phases of plain top-p.
//
// Performance notes: every pass over the 128k logits is L2-latency bound, so logits are read 128 bits at a time
// (two loads in flight per thread on plain rows); histogram mass is accumulated in 32.32 fixed point with native
// 32-bit shared-memory atomics (float / 64-bit shared atomics are CAS loops).
#include "kernels.h"

#include "common.cuh"
#include "launch.cuh"

namespace b2b {

constexpr int SAMP_THREADS = 1024;

__device__ __forceinline__ uint32_t hash_u32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  return x;
}

// logit -> (soft-cap) -> (+ bias b) -> repetition penalty -> (presence / frequency penalty) -> temperature, with the
// bias and count steps compiled in only for the row kinds that read them
template <bool BIAS, bool COUNTS>
__device__ __forceinline__ float transform(float l, float b, bool is_seen, int c, float pen, float pres, float freq,
                                           float inv_temp, float cap) {
  if (cap > 0.f) l = cap * tanhf(l / cap);
  if constexpr (BIAS) l = __fadd_rn(l, b);
  if (is_seen) l = l > 0.f ? l / pen : l * pen;
  if constexpr (COUNTS) {
    if (c > 0) l = __fsub_rn(__fsub_rn(l, __fmul_rn(freq, static_cast<float>(c))), pres);
  }
  return l * inv_temp;
}

// phase-1 row kinds, chosen per row (see phase 1 in sample_kernel)
enum RowKind { ROW_PLAIN, ROW_COUNTED, ROW_BIASED };
template <RowKind K>
struct Row { static constexpr RowKind value = K; };

// butterfly max / argmax over the warp; on equal values the lower id wins.  The test has no short-circuit, so that it
// compiles to selects rather than branches.
__device__ __forceinline__ void warp_argmax(float& mx, int& amx) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, mx, o);
    const int oi = __shfl_xor_sync(0xffffffffu, amx, o);
    if ((om > mx) | ((om == mx) & (oi < amx))) { mx = om; amx = oi; }
  }
}
template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// inclusive prefix sum over the lanes of the warp
template <typename T>
__device__ __forceinline__ T warp_scan(T v, int lane) {
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const T t = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += t; }
  return v;
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
  unsigned long long czk[MAX_CS];           // per-CTA partials of Z_K, the mass of the top-k set
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
// histogram kind for merge_and_find: 32.32 fixed-point mass in two words, or a 32-bit token count in one
template <bool C>
struct CountHist { static constexpr bool value = C; };

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
  const float pres = p.presence ? p.presence[bb] : 0.f;
  const float freq = p.frequency ? p.frequency[bb] : 0.f;
  const int16_t* cnt = (p.counts != nullptr && (pres != 0.f || freq != 0.f))
                           ? p.counts + static_cast<size_t>(bb) * p.cstride : nullptr;

  // exactly one thread per sequence publishes the token
  auto publish = [&](int token) {
    p.out_tokens[bb] = token;
    if (seen != nullptr) atomicOr(&seen[token >> 5], 1u << (token & 31));
    if (p.counts != nullptr) {
      int16_t* c = p.counts + static_cast<size_t>(bb) * p.cstride + token;
      const int16_t v = *c;
      if (v < 32767) *c = static_cast<int16_t>(v + 1);
    }
    if (p.history != nullptr) {
      const int pos = p.hist_pos[bb];
      // the history is a ring: the host reads each burst's window before the writer can lap it
      p.history[static_cast<size_t>(bb) * p.hist_stride + (pos % p.hist_stride)] = token;
      p.hist_pos_out[bb] = pos + 1;
    }
    if (p.peer_tokens != nullptr && p.peer_tokens != p.out_tokens) p.peer_tokens[bb] = token;
    arrive();
  };

  const int nbias = p.bias_n ? min(p.bias_n[bb], p.bias_stride) : 0;

  // ---- phase 1: L2 -> transform() -> shared memory, with a running max / argmax.  Each thread visits its ids in
  // increasing order and keeps the first maximum, so ties go to the lowest id.  The row kind is uniform per row and
  // decides which steps of transform() are compiled in and what the pass reads beside the logits and `seen`:
  //   * biased (nbias > 0): the bias staged in the ebuf slot that the transformed logit then overwrites, and the
  //     counts when cnt != nullptr; one quad (4 ids) per thread per iteration;
  //   * counted (cnt != nullptr): the 4 counts of a quad in one aligned 8-byte load; one quad per iteration;
  //   * plain: two quads per iteration, so two 128-bit loads are in flight.
  float mx = -INFINITY; int amx = 0;
  auto phase1 = [&](auto kind) {
    constexpr RowKind K = decltype(kind)::value;
    constexpr bool BIAS = K == ROW_BIASED;
    constexpr int Q = K == ROW_PLAIN ? 2 : 1;                 // quads per thread per iteration
    const bool has_cnt = K == ROW_COUNTED || (BIAS && cnt != nullptr);
    auto take = [&](int i, float raw, float bias, uint32_t sw, int c) {
      const float l = transform<BIAS, K != ROW_PLAIN>(raw, bias, (sw >> (i & 31)) & 1u, c, pen, pres, freq, inv_temp,
                                                      cap);
      ebuf[i - lo] = l;
      if (l > mx) { mx = l; amx = i; }
    };
    for (int q = tid; q < n4; q += Q * SAMP_THREADS) {
      float a[Q][4] = {};
      // vec_ok outermost: the 128-bit loads of all Q quads issue back to back
      if (vec_ok) {
#pragma unroll
        for (int u = 0; u < Q; ++u) {
          if (u > 0 && q + u * SAMP_THREADS >= n4) break;
          const int i0 = lo + 4 * (q + u * SAMP_THREADS);
          const float4 va = *reinterpret_cast<const float4*>(logits + i0);
          a[u][0] = va.x; a[u][1] = va.y; a[u][2] = va.z; a[u][3] = va.w;
        }
      } else {
#pragma unroll
        for (int u = 0; u < Q; ++u) {
          if (u > 0 && q + u * SAMP_THREADS >= n4) break;
          const int i0 = lo + 4 * (q + u * SAMP_THREADS);
#pragma unroll
          for (int k = 0; k < 4; ++k) a[u][k] = logits[i0 + k];
        }
      }
#pragma unroll
      for (int u = 0; u < Q; ++u) {
        const int qu = q + u * SAMP_THREADS, i0 = lo + 4 * qu;
        if (u > 0 && qu >= n4) break;
        const float4 bv = BIAS ? reinterpret_cast<const float4*>(ebuf)[qu] : make_float4(0.f, 0.f, 0.f, 0.f);
        const uint2 cw = has_cnt ? *reinterpret_cast<const uint2*>(cnt + i0) : make_uint2(0u, 0u);
        const uint32_t sw = seen_r ? seen_r[i0 >> 5] : 0u;
        take(i0, a[u][0], bv.x, sw, static_cast<int16_t>(cw.x & 0xFFFFu));
        take(i0 + 1, a[u][1], bv.y, sw, static_cast<int16_t>(cw.x >> 16));
        take(i0 + 2, a[u][2], bv.z, sw, static_cast<int16_t>(cw.y & 0xFFFFu));
        take(i0 + 3, a[u][3], bv.w, sw, static_cast<int16_t>(cw.y >> 16));
      }
    }
    for (int i = lo + 4 * n4 + tid; i < hi; i += SAMP_THREADS)
      take(i, logits[i], BIAS ? ebuf[i - lo] : 0.f, seen_r ? seen_r[i >> 5] : 0u, has_cnt ? cnt[i] : 0);
  };
  if (nbias > 0) {
    // stage the bias of the ids this CTA owns in its slice (0 for the others)
    for (int j = tid; j < n; j += SAMP_THREADS) ebuf[j] = 0.f;
    __syncthreads();
    const size_t row = static_cast<size_t>(bb) * p.bias_stride;
    for (int j = tid; j < nbias; j += SAMP_THREADS) {
      const int id = p.bias_ids[row + j];
      if (id >= lo && id < hi) ebuf[id - lo] = p.bias_vals[row + j];
    }
    __syncthreads();
    phase1(Row<ROW_BIASED>{});
  } else if (cnt != nullptr) {
    phase1(Row<ROW_COUNTED>{});
  } else {
    phase1(Row<ROW_PLAIN>{});
  }
  warp_argmax(mx, amx);
  if (lane == 0) { S.red_f[warp] = mx; S.red_i[warp] = amx; }
  __syncthreads();
  cluster_wait_acquire();            // all CTAs of the cluster are running (pairs with the arrive at kernel entry)
  if (warp == 0) {
    mx = S.red_f[lane]; amx = S.red_i[lane];
    warp_argmax(mx, amx);
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

  // sum of v over the cluster: each CTA's total goes to slot[r] of every CTA, and after the cluster barrier each CTA
  // adds the CS slots in rank order, so all of them get the same sum
  auto cluster_total = [&](unsigned long long v, unsigned long long* slot) {
    v = warp_sum(v);
    if (lane == 0) S.red_u[warp] = v;
    __syncthreads();
    if (warp == 0) {
      const unsigned long long z = warp_sum(S.red_u[lane]);
      if (lane < CS) st_dsmem_u64(mapa_smem(smem_u32(&slot[r]), lane), z);
    }
    cluster_sync_all();
    unsigned long long t = 0ull;
    for (int c = 0; c < CS; ++c) t += slot[c];
    return t;
  };

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
  unsigned long long Z = cluster_total(zsum, S.cz);

  // cluster-wide histogram -> S.merged (every CTA computes the same sum), then a top-down search for the
  // highest bin whose suffix mass (plus `carry`) reaches `need`.  Results: s_i[0] = bin, s_u[0] = mass above it.
  // `kind` is CountHist<true> for a count histogram in `hlo` alone (then the suffix is a token count).
  auto merge_and_find = [&](auto kind, const uint32_t* hlo, const uint32_t* hhi, unsigned long long carry,
                            unsigned long long need) {
    {
      const int bin = 2 * tid;        // SBINS == 2 * SAMP_THREADS
      unsigned long long m0 = 0ull, m1 = 0ull;
      const uint32_t alo = smem_u32(&hlo[bin]);
      for (int c = 0; c < CS; ++c) {
        const uint2 l2 = ld_dsmem_v2u32(mapa_smem(alo, c));
        if constexpr (decltype(kind)::value) {
          m0 += l2.x;
          m1 += l2.y;
        } else {
          const uint2 h2 = ld_dsmem_v2u32(mapa_smem(smem_u32(&hhi[bin]), c));
          m0 += (static_cast<unsigned long long>(h2.x) << 32) | l2.x;
          m1 += (static_cast<unsigned long long>(h2.y) << 32) | l2.y;
        }
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
      const unsigned long long pre = warp_scan(v, lane);
      const unsigned ball = __ballot_sync(0xffffffffu, carry + pre >= need);
      int found = -1;
      unsigned long long above = carry;
      if (ball) {
        const int l0 = __ffs(ball) - 1;
        unsigned long long run = carry + __shfl_sync(0xffffffffu, pre, l0) - __shfl_sync(0xffffffffu, v, l0);
        const int cbase = (31 - l0) * 64;
        for (int base = cbase + 32; base >= cbase && found < 0; base -= 32) {
          const unsigned long long bv = S.merged[base + (31 - lane)];
          const unsigned long long bp = warp_scan(bv, lane);
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

  // ---- top-k (row-uniform): the 22-bit key prefix thr_k of the k-th largest e from two count levels, then
  // Z = Z_K, the mass of {key >= thr_k}.  The level-2 arrays are idle until phase 3 and hold the counts.
  const int top_k = p.top_k ? p.top_k[bb] : 0;
  if (top_k > 0 && top_k < V) {
    for (int j = tid; j < n; j += SAMP_THREADS) atomicAdd(&S.h2_lo[dkey(ebuf[j]) >> 17], 1u);
    __syncthreads();
    cluster_sync_all();
    merge_and_find(CountHist<true>{}, S.h2_lo, nullptr, 0ull, static_cast<unsigned long long>(top_k));
    const int K1 = S.s_i[0];
    const unsigned long long above_k = S.s_u[0];      // tokens strictly above the boundary bin
    __syncthreads();
    for (int j = tid; j < n; j += SAMP_THREADS) {
      const uint32_t d = dkey(ebuf[j]);
      if (static_cast<int>(d >> 17) == K1) atomicAdd(&S.h2_hi[(d >> 6) & (SBINS - 1)], 1u);
    }
    __syncthreads();
    cluster_sync_all();
    merge_and_find(CountHist<true>{}, S.h2_hi, nullptr, above_k, static_cast<unsigned long long>(top_k));
    const uint32_t thr_k = (static_cast<uint32_t>(K1) << 17) | (static_cast<uint32_t>(S.s_i[0]) << 6);
    unsigned long long zk = 0ull;
    for (int j = tid; j < n; j += SAMP_THREADS) {
      const float e = ebuf[j];
      if (dkey(e) >= thr_k) zk += fx32(e);
    }
    Z = cluster_total(zk, S.czk);     // its cluster barrier also ends every peer's reads of the count histograms
    for (int i = tid; i < SBINS; i += SAMP_THREADS) { S.h2_lo[i] = 0u; S.h2_hi[i] = 0u; }
    // the __syncthreads inside the level-1 search below orders these stores before phase 3
  }

  const unsigned long long need = static_cast<unsigned long long>(static_cast<double>(top_p) * static_cast<double>(Z));
  merge_and_find(CountHist<false>{}, S.h1_lo, S.h1_hi, 0ull, need);
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
  merge_and_find(CountHist<false>{}, S.h2_lo, S.h2_hi, above1, need);
  // the nucleus is a prefix of K (need <= Z_K), so thr >= thr_k; min-p (row-uniform) can only raise it
  uint32_t thr = (static_cast<uint32_t>(B1) << 17) | (static_cast<uint32_t>(S.s_i[0]) << 6);
  const float min_p = p.min_p ? p.min_p[bb] : 0.f;
  if (min_p > 0.f) thr = max(thr, dkey(fminf(min_p, 1.f)));

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
  mine = warp_sum(mine);
  if (lane == 0) S.wtot[warp] = mine;
  __syncthreads();
  // inclusive prefix over the 32 warp totals (every warp computes the same values)
  const float wt = S.wtot[lane];
  const float wpre = warp_scan(wt, lane);
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
    const float pre = warp_scan(v, lane);
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

int launch_sample(const SampleParams& p, int batch, cudaStream_t s) {
  const int vocab = p.vocab;
  if (p.counts != nullptr && (p.cstride < vocab || p.cstride % 8 != 0 ||
                              (reinterpret_cast<uintptr_t>(p.counts) & 7) != 0))
    return -7;
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
