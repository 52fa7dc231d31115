// Paged-KV attention for sm_90a (decode + chunked prefill), GQA-aware.
//
// One CTA = (sequence, kv head, query block [, kv split]).  All G = n_q/n_kv query
// heads that share the kv head are processed together, so each K/V page is read from
// HBM exactly once per group (the op is KV-bandwidth bound at decode).  K/V pages are
// staged into padded shared memory with cp.async (double buffered), scores use an
// online softmax in fp32.  Supports sliding windows (Mistral / Gemma-2 local layers),
// logit soft-capping (Gemma-2) and split-KV with a merge pass for long contexts.
//
// Layouts: q [tokens, n_q, D] (pre-scaled by 1/sqrt(D), rotary applied by the QKV GEMM
// epilogue), K/V cache [pages, 64, n_kv, D], block_table [seqs, max_pages].
// Reference parity: torch SDPA + HF DynamicCache under bee2bee/hf.py:42-43.
#include "kernels.h"

#include "common.cuh"
#include "launch.cuh"

namespace b2b {

constexpr int PAGE = 64;          // tokens per KV page == tokens per smem tile
constexpr int ATT_THREADS = 128;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

struct AttnParams {
  const __nv_bfloat16* q;       // [tokens, n_q, D]
  const __nv_bfloat16* k_cache; // [pages, PAGE, n_kv, D]
  const __nv_bfloat16* v_cache;
  __nv_bfloat16* out;           // [tokens, n_q, D]
  const int* block_table;       // [seqs, max_pages]
  const int* q_start;           // [seqs] first query token of the sequence in q/out
  const int* q_len;             // [seqs]
  const int* kv_len;            // [seqs] total kv length including the new tokens
  float* ws;                    // split workspace [seqs, n_kv, splits, R, D+2] (decode only)
  int max_pages, n_q, n_kv, window, splits;
  float softcap;
};

// R = query rows per CTA (G * QB, padded to a multiple of 4), D = head dim
template <int D, int R>
__global__ void __launch_bounds__(ATT_THREADS) attn_kernel(const AttnParams p, const int G, const int QB) {
  pdl_launch_dependents();
  pdl_wait();
  constexpr int DP = D + 8;                      // padded row (bf16) -> conflict-free 16B reads
  extern __shared__ __align__(16) uint8_t smem_raw[];
  __nv_bfloat16* k_s = reinterpret_cast<__nv_bfloat16*>(smem_raw);            // [2][PAGE][DP]
  __nv_bfloat16* v_s = k_s + 2 * PAGE * DP;                                    // [2][PAGE][DP]
  float* q_s = reinterpret_cast<float*>(v_s + 2 * PAGE * DP);                  // [R][D]
  float* p_s = q_s + R * D;                                                    // [R][PAGE]
  float* m_s = p_s + R * PAGE;                                                 // [R] running max
  float* l_s = m_s + R;                                                        // [R] running sum
  float* a_s = l_s + R;                                                        // [R] rescale factor

  const int seq = blockIdx.z, kvh = blockIdx.y;
  const int split = (p.splits > 1) ? blockIdx.x : 0;
  const int qblk = (p.splits > 1) ? 0 : blockIdx.x;
  const int qlen = p.q_len[seq], kvlen = p.kv_len[seq];
  const int q0 = qblk * QB;
  if (q0 >= qlen) return;
  const int nq_here = min(QB, qlen - q0);
  const int qtok0 = p.q_start[seq] + q0;
  const int pos0 = kvlen - qlen + q0;            // absolute position of query row 0
  const int tid = threadIdx.x;

  // row r -> (query i = r / G, head g = r % G)
  for (int idx = tid; idx < R * D; idx += ATT_THREADS) {
    const int r = idx / D, d = idx % D;
    const int i = r / G, g = r % G;
    float v = 0.f;
    if (i < nq_here && r < G * QB)
      v = __bfloat162float(p.q[(static_cast<size_t>(qtok0 + i) * p.n_q + kvh * G + g) * D + d]);
    q_s[idx] = v;
  }
  if (tid < R) { m_s[tid] = -INFINITY; l_s[tid] = 0.f; a_s[tid] = 1.f; }
  __syncthreads();

  // kv range visible to this CTA
  int kv_hi = min(kvlen, pos0 + nq_here);                       // causal upper bound (exclusive)
  int kv_lo = 0;
  if (p.window > 0) kv_lo = max(0, pos0 - p.window + 1);
  int t_lo = kv_lo / PAGE, t_hi = (kv_hi + PAGE - 1) / PAGE;    // page-tile range
  if (p.splits > 1) {
    const int nt = t_hi - t_lo;
    const int a = t_lo + (nt * split) / p.splits, b = t_lo + (nt * (split + 1)) / p.splits;
    t_lo = a; t_hi = b;
  }

  const int* bt = p.block_table + static_cast<size_t>(seq) * p.max_pages;
  auto issue_tile = [&](int t, int buf) {
    const int page = bt[t];
    const __nv_bfloat16* kg = p.k_cache + (static_cast<size_t>(page) * PAGE * p.n_kv + kvh) * D;
    const __nv_bfloat16* vg = p.v_cache + (static_cast<size_t>(page) * PAGE * p.n_kv + kvh) * D;
    constexpr int CH = D / 8;                     // 16B chunks per row
    for (int c = tid; c < PAGE * CH; c += ATT_THREADS) {
      const int row = c / CH, ch = c % CH;
      cp_async16(k_s + (buf * PAGE + row) * DP + ch * 8, kg + static_cast<size_t>(row) * p.n_kv * D + ch * 8);
      cp_async16(v_s + (buf * PAGE + row) * DP + ch * 8, vg + static_cast<size_t>(row) * p.n_kv * D + ch * 8);
    }
    cp_async_commit();
  };

  // PV accumulators: warp w owns rows [w*R/4, (w+1)*R/4), lane owns D/32 contiguous dims
  constexpr int RW = R / 4, DL = D / 32;
  float acc[RW][DL];
#pragma unroll
  for (int a = 0; a < RW; ++a)
#pragma unroll
    for (int b = 0; b < DL; ++b) acc[a][b] = 0.f;
  const int warp = tid >> 5, lane = tid & 31;

  if (t_lo < t_hi) issue_tile(t_lo, 0);
  for (int t = t_lo; t < t_hi; ++t) {
    const int buf = (t - t_lo) & 1;
    if (t + 1 < t_hi) { issue_tile(t + 1, buf ^ 1); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
    __syncthreads();

    // ---- S = q K^T : thread -> (token j = tid % 64, row half = tid / 64)
    {
      constexpr int RH = R / 2;
      const int j = tid & 63, rh = tid >> 6;
      float s[RH];
#pragma unroll
      for (int a = 0; a < RH; ++a) s[a] = 0.f;
      const __nv_bfloat16* krow = k_s + (buf * PAGE + j) * DP;
#pragma unroll 4
      for (int d0 = 0; d0 < D; d0 += 8) {
        uint4 kv = *reinterpret_cast<const uint4*>(krow + d0);
        const __nv_bfloat162* kh = reinterpret_cast<const __nv_bfloat162*>(&kv);
        float kf[8];
#pragma unroll
        for (int e = 0; e < 4; ++e) { float2 f = __bfloat1622float2(kh[e]); kf[2 * e] = f.x; kf[2 * e + 1] = f.y; }
#pragma unroll
        for (int a = 0; a < RH; ++a) {
          const float4* qp = reinterpret_cast<const float4*>(q_s + (rh * RH + a) * D + d0);
          const float4 qa = qp[0], qb = qp[1];
          s[a] += qa.x * kf[0] + qa.y * kf[1] + qa.z * kf[2] + qa.w * kf[3] + qb.x * kf[4] + qb.y * kf[5] +
                  qb.z * kf[6] + qb.w * kf[7];
        }
      }
      const int kvpos = t * PAGE + j;
#pragma unroll
      for (int a = 0; a < RH; ++a) {
        const int r = rh * RH + a;
        const int qpos = pos0 + r / G;
        float v = s[a];
        if (p.softcap > 0.f) v = p.softcap * tanhf(v / p.softcap);
        const bool ok = (r < G * QB) && (r / G < nq_here) && kvpos <= qpos && kvpos < kvlen &&
                        (p.window <= 0 || kvpos > qpos - p.window);
        p_s[r * PAGE + j] = ok ? v : -INFINITY;
      }
    }
    __syncthreads();

    // ---- online softmax per row (one warp handles R/4 rows, 64 columns each)
    for (int a = 0; a < RW; ++a) {
      const int r = warp * RW + a;
      const float x0 = p_s[r * PAGE + lane], x1 = p_s[r * PAGE + lane + 32];
      float mx = fmaxf(x0, x1);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      const float m_old = m_s[r];
      const float m_new = fmaxf(m_old, mx);
      const float e0 = (m_new == -INFINITY) ? 0.f : __expf(x0 - m_new);
      const float e1 = (m_new == -INFINITY) ? 0.f : __expf(x1 - m_new);
      float sum = e0 + e1;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      const float alpha = (m_new == -INFINITY) ? 1.f : __expf(m_old - m_new);
      p_s[r * PAGE + lane] = e0;
      p_s[r * PAGE + lane + 32] = e1;
      if (lane == 0) { m_s[r] = m_new; l_s[r] = l_s[r] * alpha + sum; a_s[r] = alpha; }
    }
    __syncwarp();

    // ---- O += P V : warp -> its RW rows, lane -> DL dims   (p_s rows are warp-private here)
    {
#pragma unroll
      for (int a = 0; a < RW; ++a) {
        const float alpha = a_s[warp * RW + a];
#pragma unroll
        for (int b = 0; b < DL; ++b) acc[a][b] *= alpha;
      }
      const __nv_bfloat16* vbase = v_s + buf * PAGE * DP + lane * DL;
#pragma unroll 4
      for (int j = 0; j < PAGE; ++j) {
        float vf[DL];
        if constexpr (DL == 4) {
          uint2 raw = *reinterpret_cast<const uint2*>(vbase + j * DP);
          const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
          float2 f0 = __bfloat1622float2(h[0]), f1 = __bfloat1622float2(h[1]);
          vf[0] = f0.x; vf[1] = f0.y; vf[2] = f1.x; vf[3] = f1.y;
        } else if constexpr (DL == 8) {
          uint4 raw = *reinterpret_cast<const uint4*>(vbase + j * DP);
          const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&raw);
#pragma unroll
          for (int e = 0; e < 4; ++e) { float2 f = __bfloat1622float2(h[e]); vf[2 * e] = f.x; vf[2 * e + 1] = f.y; }
        } else {
          const __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162*>(vbase + j * DP);
          float2 f = __bfloat1622float2(h);
          vf[0] = f.x; vf[1] = f.y;
        }
#pragma unroll
        for (int a = 0; a < RW; ++a) {
          const float pj = p_s[(warp * RW + a) * PAGE + j];
#pragma unroll
          for (int b = 0; b < DL; ++b) acc[a][b] += pj * vf[b];
        }
      }
    }
    __syncthreads();
  }

  // ---- finalize
#pragma unroll
  for (int a = 0; a < RW; ++a) {
    const int r = warp * RW + a;
    const int i = r / G, g = r % G;
    if (r >= G * QB || i >= nq_here) continue;
    const float l = l_s[r], m = m_s[r];
    if (p.splits > 1) {
      float* w = p.ws + (((static_cast<size_t>(seq) * p.n_kv + kvh) * p.splits + split) * R + r) * (D + 2);
#pragma unroll
      for (int b = 0; b < DL; ++b) w[lane * DL + b] = acc[a][b];
      if (lane == 0) { w[D] = m; w[D + 1] = l; }
    } else {
      const float inv = l > 0.f ? 1.f / l : 0.f;
      __nv_bfloat16* o = p.out + (static_cast<size_t>(qtok0 + i) * p.n_q + kvh * G + g) * D + lane * DL;
#pragma unroll
      for (int b = 0; b < DL; ++b) o[b] = __float2bfloat16_rn(acc[a][b] * inv);
    }
  }
}

// merge split partials: grid (seqs, n_kv), block = R*32 threads? -> one warp per row
template <int D, int R>
__global__ void attn_merge_kernel(const AttnParams p, const int G) {
  pdl_launch_dependents();
  pdl_wait();
  const int seq = blockIdx.x, kvh = blockIdx.y;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // an inactive sequence (q_len 0) has no partials (its split CTAs return at once) and no output row of its own
  if (warp >= G || p.q_len[seq] <= 0) return;
  const int r = warp;                       // decode: QB = 1 -> row == head in group
  constexpr int DL = D / 32;
  float m = -INFINITY;
  const float* base = p.ws + ((static_cast<size_t>(seq) * p.n_kv + kvh) * p.splits) * R * (D + 2);
  for (int s = 0; s < p.splits; ++s) m = fmaxf(m, base[(static_cast<size_t>(s) * R + r) * (D + 2) + D]);
  float acc[DL];
#pragma unroll
  for (int b = 0; b < DL; ++b) acc[b] = 0.f;
  float l = 0.f;
  for (int s = 0; s < p.splits; ++s) {
    const float* w = base + (static_cast<size_t>(s) * R + r) * (D + 2);
    const float ms = w[D];
    const float sc = (ms == -INFINITY) ? 0.f : __expf(ms - m);
    l += w[D + 1] * sc;
#pragma unroll
    for (int b = 0; b < DL; ++b) acc[b] += w[lane * DL + b] * sc;
  }
  const float inv = l > 0.f ? 1.f / l : 0.f;
  const int tok = p.q_start[seq];
  __nv_bfloat16* o = p.out + (static_cast<size_t>(tok) * p.n_q + kvh * G + r) * D + lane * DL;
#pragma unroll
  for (int b = 0; b < DL; ++b) o[b] = __float2bfloat16_rn(acc[b] * inv);
}

template <int D, int R>
static int launch_attn_t(const AttnParams& p, int G, int QB, int seqs, int max_qblocks, cudaStream_t s) {
  constexpr int DP = D + 8;
  const int smem = 4 * PAGE * DP * 2 + (R * D + R * PAGE + 3 * R) * 4;
  static bool set = false;
  if (!set) {
    cudaError_t e = cudaFuncSetAttribute(attn_kernel<D, R>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return static_cast<int>(e);
    set = true;
  }
  dim3 grid(p.splits > 1 ? p.splits : max_qblocks, p.n_kv, seqs);
  cudaError_t e = launch_kernel(attn_kernel<D, R>, grid, dim3(ATT_THREADS), smem, s, 1, p, G, QB);
  if (e != cudaSuccess) return static_cast<int>(e);
  if (p.splits > 1) {
    e = launch_kernel(attn_merge_kernel<D, R>, dim3(seqs, p.n_kv), dim3(32 * (G < 1 ? 1 : G)), 0, s, 1, p, G);
  }
  return static_cast<int>(e);
}

template <int D, int R>
static int attn_set_attr() {
  constexpr int DP = D + 8;
  const int smem = 4 * PAGE * DP * 2 + (R * D + R * PAGE + 3 * R) * 4;
  return static_cast<int>(cudaFuncSetAttribute(attn_kernel<D, R>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
}
int attention_init() {
  int r = 0;
#define B2B_ATT_INIT(DD, RR) if ((r = attn_set_attr<DD, RR>())) return r;
  B2B_ATT_INIT(64, 4) B2B_ATT_INIT(64, 8) B2B_ATT_INIT(64, 16) B2B_ATT_INIT(64, 32) B2B_ATT_INIT(64, 64)
  B2B_ATT_INIT(128, 4) B2B_ATT_INIT(128, 8) B2B_ATT_INIT(128, 16) B2B_ATT_INIT(128, 32) B2B_ATT_INIT(128, 64)
  B2B_ATT_INIT(256, 4) B2B_ATT_INIT(256, 8) B2B_ATT_INIT(256, 16) B2B_ATT_INIT(256, 32)
#undef B2B_ATT_INIT
  return 0;
}

int launch_attention_merge(void* out, const int* q_start, const int* q_len, const float* ws, int seqs, int n_q, int n_kv,
                           int head_dim, int splits, cudaStream_t s) {
  AttnParams p{};
  p.out = static_cast<__nv_bfloat16*>(out);
  p.q_start = q_start;
  p.q_len = q_len;
  p.ws = const_cast<float*>(ws);
  p.n_q = n_q; p.n_kv = n_kv; p.splits = splits;
  const int G = n_q / n_kv, R = attn_rows(G, 1);
#define B2B_MERGE(DD, RR)                                                                                        \
  if (head_dim == DD && R == RR)                                                                                  \
    return static_cast<int>(launch_kernel(attn_merge_kernel<DD, RR>, dim3(seqs, n_kv), dim3(32 * (G < 1 ? 1 : G)), 0, s, 1, p, G));
  B2B_MERGE(64, 4) B2B_MERGE(64, 8) B2B_MERGE(64, 16) B2B_MERGE(128, 4) B2B_MERGE(128, 8) B2B_MERGE(128, 16)
  B2B_MERGE(256, 4) B2B_MERGE(256, 8) B2B_MERGE(256, 16)
#undef B2B_MERGE
  return -3;
}

int attn_rows(int G, int QB) {
  int r = G * QB;
  r = (r + 3) / 4 * 4;
  return r <= 4 ? 4 : (r <= 8 ? 8 : (r <= 16 ? 16 : (r <= 32 ? 32 : 64)));
}

// max_q: longest q_len in the batch (1 for decode). splits > 1 only valid when max_q == 1.
int launch_attention(const void* q, const void* k_cache, const void* v_cache, void* out, const int* block_table,
                     const int* q_start, const int* q_len, const int* kv_len, float* ws, int seqs, int max_q,
                     int max_pages, int n_q, int n_kv, int head_dim, int window, float softcap, int splits,
                     cudaStream_t s) {
  AttnParams p;
  p.q = static_cast<const __nv_bfloat16*>(q);
  p.k_cache = static_cast<const __nv_bfloat16*>(k_cache);
  p.v_cache = static_cast<const __nv_bfloat16*>(v_cache);
  p.out = static_cast<__nv_bfloat16*>(out);
  p.block_table = block_table; p.q_start = q_start; p.q_len = q_len; p.kv_len = kv_len; p.ws = ws;
  p.max_pages = max_pages; p.n_q = n_q; p.n_kv = n_kv; p.window = window; p.softcap = softcap;
  const int G = n_q / n_kv;
  if (G * n_kv != n_q || G > 16) return -2;
  if (max_q > 1) splits = 1;
  p.splits = splits < 1 ? 1 : splits;
  // query-block size: decode -> 1; prefill -> as many queries as fit 64 rows (32 for D=256)
  const int rmax = head_dim == 256 ? 32 : 64;
  int QB = 1;
  if (max_q > 1) { QB = rmax / G; if (QB < 1) QB = 1; while (QB > 1 && QB / 2 >= max_q) QB /= 2; }
  const int R = attn_rows(G, QB);
  const int max_qblocks = (max_q + QB - 1) / QB;
#define B2B_ATT(DD, RR) if (head_dim == DD && R == RR) return launch_attn_t<DD, RR>(p, G, QB, seqs, max_qblocks, s);
  B2B_ATT(64, 4) B2B_ATT(64, 8) B2B_ATT(64, 16) B2B_ATT(64, 32) B2B_ATT(64, 64)
  B2B_ATT(128, 4) B2B_ATT(128, 8) B2B_ATT(128, 16) B2B_ATT(128, 32) B2B_ATT(128, 64)
  B2B_ATT(256, 4) B2B_ATT(256, 8) B2B_ATT(256, 16) B2B_ATT(256, 32)
#undef B2B_ATT
  return -3;
}

}  // namespace b2b
