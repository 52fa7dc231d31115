// Prefill (and chunked-prefill) attention on the Hopper tensor cores: flash-attention forward over the paged KV
// cache with wgmma, accumulators in registers, operands staged by TMA.
//
// One CTA = (sequence, kv head, block of QB = 128/G queries).  The G query heads that share the kv
// head are stacked into 128 MMA rows (row = g*QB + i), so every K/V page is fetched once per
// group.  Per KV tile of BKV keys:
//     S = Q K^T      wgmma m64n64k16 (A = Q tile, B = K tile, both K-major 128B-swizzled) -> registers
//     P = softmax    online max with lazy rescaling, on the accumulator fragment (four threads per row)
//     O += P V       wgmma m64nDk16 (A = P from registers as bf16, B = V tile read MN-major:
//                                    the cache keeps V as [token, d], i.e. N-contiguous)
// Warp roles: 0..7 = two consumer warpgroups (rows 0..63 / 64..127), 8 = TMA producer.
// q is pre-scaled by 1/sqrt(d) and rotated by the QKV GEMM epilogue; K is rotated when appended.
//
// Layouts: q/out [tokens, n_q, D]; K/V cache [pages, 64, n_kv, D]; block_table [seqs, max_pages].
// Reference parity: torch SDPA under `transformers.generate` (bee2bee/hf.py:42-43).
#include "kernels.h"

#include <cuda.h>
#include <cuda_fp8.h>

#include <cstdlib>
#include <type_traits>

#include "common.cuh"
#include "launch.cuh"
#include "wgmma.cuh"

namespace b2b {

int make_tmap_shared(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint64_t ld, uint32_t box_rows,
                     int elt_bytes);

namespace {

constexpr int APAGE = 64;
constexpr int ATC_CONSUMERS = 256;                 // two warpgroups of 64 query rows
constexpr int ATC_THREADS = ATC_CONSUMERS + 32;     // + TMA producer warp
constexpr float LOG2E = 1.4426950408889634f;

struct AttnTcParams {
  __nv_bfloat16* out;
  const int* block_table;
  const int* q_start;
  const int* q_len;
  const int* kv_len;
  int max_pages, n_q, n_kv, window;
  float softcap;
  // split-KV decode (q_len == 1): grid.x = splits, CTA `split` covers a contiguous range of the 64-key tiles and writes
  // its unnormalised partial (O, running max, row sum) to the workspace the CUDA-core kernel's merge pass reads:
  // ws[((seq * n_kv + kvh) * splits + split) * ws_rows + head_in_group][D + 2]
  int splits, ws_rows;
  float* ws;
  // fused MX quantisation of the output for the O-proj GEMM (mxfp8 pieces): the four threads of a row own a 32-feature
  // block together, so the block maximum is a two-step shuffle: e4m3 bytes + UE8M0 scale in the consumer's scale-factor
  // chunk layout (token tile q_bn).  Not available in split-KV mode (the merge pass writes the output).
  uint8_t* q_out8;
  uint8_t* q_sf;
  int q_bn;
};

template <int D>
struct AtcCfg {
  static constexpr int BKV = 64;                                  // keys per tile == one KV page
  static constexpr int kQBytes = 128 * D * 2;
  static constexpr int kKVBytes = BKV * D * 2;
  static constexpr int kSmemBytes = kQBytes + 4 * kKVBytes + 256;
};

template <int D, bool SOFTCAP>
__global__ void __launch_bounds__(ATC_THREADS, 1)
attn_prefill_tc_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_k,
                       const __grid_constant__ CUtensorMap tm_v, const AttnTcParams p, const int G, const int QB) {
  using Cfg = AtcCfg<D>;
  constexpr int BKV = Cfg::BKV;
  constexpr int DB = D / 64;            // 64-column (128 B) blocks of the head dim

  // ---- set-up that reads nothing an earlier kernel wrote (barriers, descriptor prefetch): under PDL the CTA is
  // resident while the QKV GEMM still drains, so all of this is off the critical path; only then wait for the producer
  extern __shared__ __align__(1024) uint8_t smem[];
  if ((smem_u32(smem) & 1023u) != 0u) __trap();             // the swizzled tiles need 1024-byte alignment
  uint8_t* q_s = smem;
  uint8_t* k_s = q_s + Cfg::kQBytes;                       // [2][kKVBytes]
  uint8_t* v_s = k_s + 2 * Cfg::kKVBytes;                  // [2][kKVBytes]
  uint64_t* bars = reinterpret_cast<uint64_t*>(v_s + 2 * Cfg::kKVBytes);
  uint64_t* q_full = bars + 0;
  uint64_t* k_full = bars + 1;     // [2]
  uint64_t* v_full = bars + 3;     // [2]
  uint64_t* k_empty = bars + 5;    // [2]
  uint64_t* v_empty = bars + 7;    // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == ATC_CONSUMERS) {
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&k_full[i], 1); mbar_init(&v_full[i], 1);
      mbar_init(&k_empty[i], ATC_CONSUMERS / 32); mbar_init(&v_empty[i], ATC_CONSUMERS / 32);
    }
    fence_barrier_init();
    tma_prefetch_desc(&tm_q); tma_prefetch_desc(&tm_k); tma_prefetch_desc(&tm_v);
  }
  __syncthreads();

  pdl_launch_dependents();                                  // dependents (the O-proj GEMM) may become resident
  pdl_wait();                                               // q / K / V and the metadata below come from earlier kernels
  const int seq = blockIdx.z, kvh = blockIdx.y;
  const bool split_mode = p.splits > 1;
  const int qblk = split_mode ? 0 : gridDim.x - 1 - blockIdx.x;   // longest (latest) query blocks first
  const int qlen = p.q_len[seq], kvlen = p.kv_len[seq];
  const int q0 = qblk * QB;
  bool active = q0 < qlen;                                  // CTA-uniform; an idle CTA returns at once
  const int nq_here = min(QB, qlen - q0);
  const int qtok0 = p.q_start[seq] + q0;
  const int pos0 = kvlen - qlen + q0;                       // absolute position of query 0 of this block
  const int kv_hi = min(kvlen, pos0 + nq_here);
  const int kv_lo = p.window > 0 ? max(0, pos0 - p.window + 1) : 0;
  int t_lo = kv_lo / BKV, t_hi = (kv_hi + BKV - 1) / BKV;
  if (active && split_mode) {
    // this CTA's share of the key tiles (may be empty: it then publishes an empty partial, m = -inf, l = 0)
    const int per = (t_hi - t_lo + p.splits - 1) / p.splits;
    t_lo = min(t_hi, t_lo + static_cast<int>(blockIdx.x) * per);
    t_hi = min(t_hi, t_lo + per);
    if (t_hi <= t_lo) {
      // empty share (short sequence, many splits): publish an empty partial; no TMA / MMA is ever issued by this CTA
      if (threadIdx.x < G) {
        float* w = p.ws + (((static_cast<size_t>(seq) * p.n_kv + kvh) * p.splits + blockIdx.x) * p.ws_rows + threadIdx.x) * (D + 2);
        for (int c = 0; c < D; ++c) w[c] = 0.f;
        w[D] = -INFINITY;
        w[D + 1] = 0.f;
      }
      active = false;
    }
  }
  const int nt = t_hi - t_lo;
  if (!active) return;

  if (warp == ATC_CONSUMERS / 32) {
    // ------------------------------------------------------------------ TMA producer
    if (lane == 0) {
      mbar_arrive_expect_tx(q_full, Cfg::kQBytes);
      for (int g = 0; g < G; ++g)
        for (int c = 0; c < DB; ++c)
          tma_load_2d(q_s + c * (128 * 128) + g * QB * 128, &tm_q, q_full, (kvh * G + g) * D + c * 64, qtok0);
      const int* bt = p.block_table + static_cast<size_t>(seq) * p.max_pages;
      for (int n = 0; n < nt; ++n) {
        const int s = n & 1;
        const uint32_t ph = static_cast<uint32_t>((n >> 1) & 1);
        const int page = bt[t_lo + n];
        mbar_wait(&k_empty[s], ph ^ 1u);
        mbar_arrive_expect_tx(&k_full[s], Cfg::kKVBytes);
#pragma unroll
        for (int c = 0; c < DB; ++c)
          tma_load_2d(k_s + s * Cfg::kKVBytes + c * (BKV * 128), &tm_k, &k_full[s], kvh * D + c * 64, page * APAGE);
        mbar_wait(&v_empty[s], ph ^ 1u);
        mbar_arrive_expect_tx(&v_full[s], Cfg::kKVBytes);
#pragma unroll
        for (int c = 0; c < DB; ++c)
          tma_load_2d(v_s + s * Cfg::kKVBytes + c * (BKV * 128), &tm_v, &v_full[s], kvh * D + c * 64, page * APAGE);
      }
    }
    return;
  }

  // ------------------------------------------------------------------ consumers: two warpgroups of 64 rows
  // wgmma fragment: this thread holds rows ra and ra + 8, columns 8j + 2*(lane % 4) (+1) of every 8-column block
  const int wg = warp >> 2;
  const int ra = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  int gq[2], iq[2], qpos[2];
  bool valid[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = ra + 8 * h;
    gq[h] = row / QB;
    iq[h] = row % QB;
    valid[h] = (gq[h] < G) && (iq[h] < nq_here);
    qpos[h] = pos0 + iq[h];
  }
  const float cap = p.softcap;
  const float inv_cap = SOFTCAP ? 1.f / cap : 0.f;
  float m_ref[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float o[D / 2];
#pragma unroll
  for (int e = 0; e < D / 2; ++e) o[e] = 0.f;
  auto release = [&](uint64_t* bar) {
    __syncwarp();
    if (lane == 0) mbar_arrive(bar);
  };

  mbar_wait(q_full, 0);
  auto tile = [&](int n, auto masked) {
    const int t = t_lo + n, s = n & 1;
    const uint32_t ph = static_cast<uint32_t>((n >> 1) & 1);
    // S = Q K^T
    float sc[BKV / 2];
#pragma unroll
    for (int e = 0; e < BKV / 2; ++e) sc[e] = 0.f;
    mbar_wait(&k_full[s], ph);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
      const uint64_t a = make_sw128_kmajor_desc(smem_u32(q_s + (kk / 4) * (128 * 128) + wg * 64 * 128)) +
                         static_cast<uint64_t>((kk % 4) * 2);
      const uint64_t b = make_sw128_kmajor_desc(smem_u32(k_s + s * Cfg::kKVBytes + (kk / 4) * (BKV * 128))) +
                         static_cast<uint64_t>((kk % 4) * 2);
      Wgmma<BKV>::bf16_ss(sc, a, b, kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(sc);
    release(&k_empty[s]);

    float mrow[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int e = 0; e < BKV / 2; ++e) {
      const int h = (e >> 1) & 1;
      float v = sc[e];
      if constexpr (SOFTCAP) v = cap * tanhf(v * inv_cap);
      v *= LOG2E;
      if constexpr (decltype(masked)::value) {
        const int kvpos = t * BKV + (e >> 2) * 8 + 2 * (lane & 3) + (e & 1);
        const bool ok = valid[h] && kvpos <= qpos[h] && kvpos < kvlen && (p.window <= 0 || kvpos > qpos[h] - p.window);
        v = ok ? v : -INFINITY;
      }
      sc[e] = v;
      mrow[h] = fmaxf(mrow[h], v);
    }
    float alpha[2], mr[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mrow[h] = fmaxf(mrow[h], __shfl_xor_sync(0xffffffffu, mrow[h], 1));
      mrow[h] = fmaxf(mrow[h], __shfl_xor_sync(0xffffffffu, mrow[h], 2));
      // lazy rescaling: keep the reference max while the new maximum is within 2^8 of it
      alpha[h] = 1.f;
      if (mrow[h] > m_ref[h] + 8.f || (m_ref[h] == -INFINITY && mrow[h] > -INFINITY)) {
        alpha[h] = (m_ref[h] == -INFINITY) ? 0.f : exp2f(m_ref[h] - mrow[h]);
        m_ref[h] = mrow[h];
      }
      mr[h] = (m_ref[h] == -INFINITY) ? 0.f : m_ref[h];          // fully masked so far: exp2(-inf - 0) = 0
    }
#pragma unroll
    for (int e = 0; e < D / 2; ++e) o[e] *= alpha[(e >> 1) & 1];
    // P = exp2(s - m_ref) -> bf16, already in the A-operand register layout of the PV wgmma
    uint32_t pa[BKV / 16][4];
    float lsum[2] = {0.f, 0.f};
#pragma unroll
    for (int e = 0; e < BKV / 2; e += 2) {
      const int h = (e >> 1) & 1;
      const float p0 = exp2f(sc[e] - mr[h]), p1 = exp2f(sc[e + 1] - mr[h]);
      lsum[h] += p0 + p1;
      const __nv_bfloat162 hv = __floats2bfloat162_rn(p0, p1);
      pa[e / 8][(e % 8) / 2] = *reinterpret_cast<const uint32_t*>(&hv);
    }
    l[0] = l[0] * alpha[0] + lsum[0];
    l[1] = l[1] * alpha[1] + lsum[1];
    // O += P V   (V tile read MN-major: the cache keeps V as [token, d], i.e. N-contiguous)
    mbar_wait(&v_full[s], ph);
    wgmma_fence_regs(o);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
      const uint64_t b = make_sw128_mnmajor_desc(smem_u32(v_s + s * Cfg::kKVBytes + kk * (16 * 128)), BKV * 128);
      Wgmma<D>::bf16_rs_tb(o, pa[kk], b, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_regs(o);
    release(&v_empty[s]);
  };

  for (int n = 0; n < nt; ++n) {
    const int t = t_lo + n;
    // a tile needs no predicate when every key of it is visible to every (valid) query row of the block
    const bool full = nq_here == QB && (t + 1) * BKV - 1 <= pos0 && (t + 1) * BKV <= kvlen &&
                      (p.window <= 0 || t * BKV > pos0 + nq_here - 1 - p.window);
    if (full) tile(n, std::false_type{}); else tile(n, std::true_type{});
  }

  // epilogue: O / l -> out[token, head, :]   (row sums: the four threads of a row each hold a quarter)
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
  }
  const int c2 = 2 * (lane & 3);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const float inv = l[h] > 0.f ? 1.f / l[h] : 0.f;
    const int tok = qtok0 + iq[h], head = kvh * G + gq[h];
    if (split_mode) {
      if (valid[h]) {
        float* wsrow = p.ws + (((static_cast<size_t>(seq) * p.n_kv + kvh) * p.splits + blockIdx.x) * p.ws_rows + gq[h]) * (D + 2);
        if ((lane & 3) == 0) {
          wsrow[D] = (m_ref[h] == -INFINITY) ? -INFINITY : m_ref[h] * 0.6931471805599453f;   // natural-log domain for the merge pass
          wsrow[D + 1] = l[h];
        }
#pragma unroll
        for (int j = 0; j < D / 8; ++j)      // rows are (D + 2) floats apart: 8-byte, not 16-byte, aligned
          *reinterpret_cast<float2*>(wsrow + 8 * j + c2) = make_float2(o[4 * j + 2 * h], o[4 * j + 2 * h + 1]);
      }
    } else if (p.q_out8 != nullptr) {
      // e4m3 + block scale of each 32 features (what a separate quantiser would compute from the bf16 output)
      const int ldq = p.n_q * D;
#pragma unroll
      for (int b = 0; b < D / 32; ++b) {
        float v[8];
        float amax = 0.f;
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          v[2 * jj] = bf16_round(o[4 * (4 * b + jj) + 2 * h] * inv);
          v[2 * jj + 1] = bf16_round(o[4 * (4 * b + jj) + 2 * h + 1] * inv);
          amax = fmaxf(amax, fmaxf(fabsf(v[2 * jj]), fabsf(v[2 * jj + 1])));
        }
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
        const uint32_t u = __float_as_uint(amax * (1.f / 448.f));
        int ex = static_cast<int>(u >> 23) - 127 + ((u & 0x7FFFFFu) ? 1 : 0);
        ex = max(-126, min(127, ex));
        const float scl = __uint_as_float(static_cast<uint32_t>(127 - ex) << 23);
        if (valid[h]) {
          const int feat = head * D + 32 * b;
          uint8_t* q8 = p.q_out8 + static_cast<size_t>(tok) * ldq + feat;
#pragma unroll
          for (int jj = 0; jj < 4; ++jj) {
            const uint16_t lo = __nv_cvt_float_to_fp8(v[2 * jj] * scl, __NV_SATFINITE, __NV_E4M3);
            const uint16_t hi = __nv_cvt_float_to_fp8(v[2 * jj + 1] * scl, __NV_SATFINITE, __NV_E4M3);
            *reinterpret_cast<uint16_t*>(q8 + 8 * jj + c2) = static_cast<uint16_t>(lo | (hi << 8));
          }
          if ((lane & 3) == 0) {
            const int tile_i = tok / p.q_bn, n = tok - tile_i * p.q_bn, rr = n & 127;
            p.q_sf[(static_cast<size_t>(tile_i) * (ldq >> 7) + (feat >> 7)) * (p.q_bn > 128 ? 1024 : 512) + (n >> 7) * 512 +
                   (rr & 31) * 16 + (rr >> 5) * 4 + ((feat >> 5) & 3)] = static_cast<uint8_t>(ex + 127);
          }
        }
      }
    } else if (valid[h]) {
      __nv_bfloat16* dst = p.out + (static_cast<size_t>(tok) * p.n_q + head) * D;
#pragma unroll
      for (int j = 0; j < D / 8; ++j)
        *reinterpret_cast<__nv_bfloat162*>(dst + 8 * j + c2) =
            __floats2bfloat162_rn(o[4 * j + 2 * h] * inv, o[4 * j + 2 * h + 1] * inv);
    }
  }
}

template <int D, bool SOFTCAP>
int launch_tc_cap(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const AttnTcParams& p, int G, int QB,
                  int seqs, int qblocks, cudaStream_t s) {
  using Cfg = AtcCfg<D>;
  static bool set[64] = {};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 64 && !set[dev]) {
    cudaError_t e = cudaFuncSetAttribute(attn_prefill_tc_kernel<D, SOFTCAP>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::kSmemBytes);
    if (e != cudaSuccess) return static_cast<int>(e);
    set[dev] = true;
  }
  return static_cast<int>(launch_kernel(attn_prefill_tc_kernel<D, SOFTCAP>,
                                        dim3(p.splits > 1 ? p.splits : qblocks, p.n_kv, seqs), dim3(ATC_THREADS),
                                        Cfg::kSmemBytes, s, 1, tq, tk, tv, p, G, QB));
}

template <int D>
int launch_tc(const CUtensorMap& tq, const CUtensorMap& tk, const CUtensorMap& tv, const AttnTcParams& p, int G, int QB,
              int seqs, int qblocks, cudaStream_t s) {
  return p.softcap > 0.f ? launch_tc_cap<D, true>(tq, tk, tv, p, G, QB, seqs, qblocks, s)
                         : launch_tc_cap<D, false>(tq, tk, tv, p, G, QB, seqs, qblocks, s);
}

}  // namespace

bool attention_tc_supported(int n_q, int n_kv, int head_dim) {
  if (n_kv <= 0 || n_q % n_kv) return false;
  const int G = n_q / n_kv;
  if (G != 1 && G != 2 && G != 4 && G != 8 && G != 16) return false;
  return head_dim == 64 || head_dim == 128 || head_dim == 256;
}

// Prefill path: every sequence contributes q_len >= 1 new tokens, kv_len includes them.
int launch_attention_tc(const void* q, const void* k_cache, const void* v_cache, void* out, const int* block_table,
                        const int* q_start, const int* q_len, const int* kv_len, int seqs, int max_q, int max_pages,
                        int n_tokens, int n_pages, int n_q, int n_kv, int head_dim, int window, float softcap,
                        int splits, float* ws, void* q_out8, void* q_sf, int q_bn, cudaStream_t s) {
  if (!attention_tc_supported(n_q, n_kv, head_dim)) return -2;
  const int G = n_q / n_kv, QB = 128 / G;
  CUtensorMap tq, tk, tv;
  int r = make_tmap_shared(&tq, q, static_cast<uint64_t>(n_tokens), static_cast<uint64_t>(n_q) * head_dim,
                           static_cast<uint64_t>(n_q) * head_dim, static_cast<uint32_t>(QB), 2);
  if (r) return r;
  const uint64_t kv_rows = static_cast<uint64_t>(n_pages) * APAGE, kv_cols = static_cast<uint64_t>(n_kv) * head_dim;
  if ((r = make_tmap_shared(&tk, k_cache, kv_rows, kv_cols, kv_cols, APAGE, 2))) return r;
  if ((r = make_tmap_shared(&tv, v_cache, kv_rows, kv_cols, kv_cols, APAGE, 2))) return r;
  AttnTcParams p;
  p.out = static_cast<__nv_bfloat16*>(out);
  p.block_table = block_table; p.q_start = q_start; p.q_len = q_len; p.kv_len = kv_len;
  p.max_pages = max_pages; p.n_q = n_q; p.n_kv = n_kv; p.window = window; p.softcap = softcap;
  p.splits = (max_q == 1 && splits > 1 && ws != nullptr) ? splits : 1;
  p.ws = ws;
  p.ws_rows = attn_rows(G, 1);
  p.q_out8 = p.splits > 1 ? nullptr : static_cast<uint8_t*>(q_out8);
  p.q_sf = static_cast<uint8_t*>(q_sf);
  p.q_bn = q_bn > 0 ? q_bn : 32;
  if (q_out8 != nullptr && p.splits > 1) return -8;       // the merge pass writes bf16: use the stand-alone quantiser
  const int qblocks = (max_q + QB - 1) / QB;
  int rc;
  switch (head_dim) {
    case 64: rc = launch_tc<64>(tq, tk, tv, p, G, QB, seqs, qblocks, s); break;
    case 128: rc = launch_tc<128>(tq, tk, tv, p, G, QB, seqs, qblocks, s); break;
    case 256: rc = launch_tc<256>(tq, tk, tv, p, G, QB, seqs, qblocks, s); break;
    default: return -3;
  }
  if (rc == 0 && p.splits > 1)
    rc = launch_attention_merge(out, q_start, q_len, ws, seqs, n_q, n_kv, head_dim, p.splits, s);
  return rc;
}

}  // namespace b2b
