// Bandwidth-bound helper kernels for sm_90a: RMSNorm / LayerNorm, embedding gather
// (optionally gated on the sampled-token flag written by the last piece over NVLink),
// KV append for the unfused path, per-token 1/rms.  All 128-bit vectorised.
// Reference parity: the ATen elementwise calls under bee2bee/hf.py:42-43.
#include "kernels.h"

#include <cuda_fp8.h>

#include "common.cuh"
#include "launch.cuh"

namespace b2b {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-wide sum for blockDim.x <= 1024
__device__ __forceinline__ float block_sum(float v, float* sh) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  float r = (threadIdx.x < nw) ? sh[threadIdx.x] : 0.f;
  if (w == 0) {
    r = warp_sum(r);
    if (l == 0) sh[0] = r;
  }
  __syncthreads();
  return sh[0];
}

// out[t] = (residual[t] +) norm(x[t]) * (gamma (+1 if gemma))   one CTA per token
__global__ void rmsnorm_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ gamma,
                               const __nv_bfloat16* __restrict__ residual, __nv_bfloat16* __restrict__ out,
                               float* __restrict__ rstd_out, int h, float eps, int gemma_plus_one) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float sh[32];
  const int t = blockIdx.x;
  const uint4* row = reinterpret_cast<const uint4*>(x + static_cast<size_t>(t) * h);
  float ss = 0.f;
  for (int i = threadIdx.x; i < h / 8; i += blockDim.x) {
    uint4 v = row[i];
    const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 f = __bfloat1622float2(p[j]);
      ss += f.x * f.x + f.y * f.y;
    }
  }
  ss = block_sum(ss, sh);
  const float rs = rsqrtf(ss / h + eps);
  if (rstd_out != nullptr && threadIdx.x == 0) rstd_out[t] = rs;
  if (out == nullptr) return;
  const uint4* grow = reinterpret_cast<const uint4*>(gamma);
  const uint4* rrow = residual ? reinterpret_cast<const uint4*>(residual + static_cast<size_t>(t) * h) : nullptr;
  uint4* orow = reinterpret_cast<uint4*>(out + static_cast<size_t>(t) * h);
  for (int i = threadIdx.x; i < h / 8; i += blockDim.x) {
    uint4 v = row[i], g = grow[i], r = rrow ? rrow[i] : make_uint4(0, 0, 0, 0), o;
    const __nv_bfloat162* pv = reinterpret_cast<const __nv_bfloat162*>(&v);
    const __nv_bfloat162* pg = reinterpret_cast<const __nv_bfloat162*>(&g);
    const __nv_bfloat162* pr = reinterpret_cast<const __nv_bfloat162*>(&r);
    __nv_bfloat162* po = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 f = __bfloat1622float2(pv[j]), gg = __bfloat1622float2(pg[j]), rr = __bfloat1622float2(pr[j]);
      if (gemma_plus_one) { gg.x += 1.f; gg.y += 1.f; }
      po[j] = __floats2bfloat162_rn(f.x * rs * gg.x + rr.x, f.y * rs * gg.y + rr.y);
    }
    orow[i] = o;
  }
}

__global__ void layernorm_kernel(const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ gamma,
                                 const __nv_bfloat16* __restrict__ beta, __nv_bfloat16* __restrict__ out, int h,
                                 float eps) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float sh[32];
  const int t = blockIdx.x;
  const __nv_bfloat16* row = x + static_cast<size_t>(t) * h;
  float s = 0.f;
  for (int i = threadIdx.x; i < h; i += blockDim.x) s += __bfloat162float(row[i]);
  const float mean = block_sum(s, sh) / h;
  float ss = 0.f;
  for (int i = threadIdx.x; i < h; i += blockDim.x) {
    float d = __bfloat162float(row[i]) - mean;
    ss += d * d;
  }
  const float rs = rsqrtf(block_sum(ss, sh) / h + eps);
  for (int i = threadIdx.x; i < h; i += blockDim.x) {
    float v = (__bfloat162float(row[i]) - mean) * rs * __bfloat162float(gamma[i]) + __bfloat162float(beta[i]);
    out[static_cast<size_t>(t) * h + i] = __float2bfloat16_rn(v);
  }
}

// out[t] = E[ids[t]] * scale (+ P[positions[t]]).  When tok_flag != null the ids were
// written by the last piece's sampler (peer store) and we acquire the flag first.
__global__ void embed_kernel(const int* __restrict__ ids, const __nv_bfloat16* __restrict__ table,
                             const __nv_bfloat16* __restrict__ pos_table, const int* __restrict__ positions,
                             __nv_bfloat16* __restrict__ out, int h, int vocab, float scale,
                             const uint32_t* tok_flag, const uint32_t* tok_epoch, const uint32_t* pf_flag,
                             const uint32_t* pf_need) {
  pdl_launch_dependents();
  pdl_wait();
  if (tok_flag != nullptr) {
    if (threadIdx.x == 0) {
      wait_flag_ge(tok_flag, *reinterpret_cast<const volatile uint32_t*>(tok_epoch) + 1);
      // decode may be enqueued right behind a prefill: the first tokens of this group's new sequences are published
      // by the last piece chunk by chunk (pf_flag counts chunks); *pf_need = chunks that must have completed
      if (pf_flag != nullptr) wait_flag_ge(pf_flag, *reinterpret_cast<const volatile uint32_t*>(pf_need));
    }
    __syncthreads();
  }
  const int t = blockIdx.x;
  int id = *reinterpret_cast<const volatile int*>(ids + t);
  id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
  const uint4* src = reinterpret_cast<const uint4*>(table + static_cast<size_t>(id) * h);
  const uint4* psrc = pos_table ? reinterpret_cast<const uint4*>(pos_table + static_cast<size_t>(positions[t]) * h) : nullptr;
  uint4* dst = reinterpret_cast<uint4*>(out + static_cast<size_t>(t) * h);
  for (int i = threadIdx.x; i < h / 8; i += blockDim.x) {
    uint4 v = src[i];
    if (scale != 1.f || psrc) {
      uint4 pp = psrc ? psrc[i] : make_uint4(0, 0, 0, 0);
      __nv_bfloat162* pv = reinterpret_cast<__nv_bfloat162*>(&v);
      const __nv_bfloat162* p2 = reinterpret_cast<const __nv_bfloat162*>(&pp);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float2 f = __bfloat1622float2(pv[j]), q = __bfloat1622float2(p2[j]);
        // HF rounds the scaled embedding to bf16 before adding anything else
        pv[j] = __floats2bfloat162_rn(bf16_round(f.x * scale) + q.x, bf16_round(f.y * scale) + q.y);
      }
    }
    dst[i] = v;
  }
}

// Unfused KV append (GPT-2 path): qkv [T, q_dim + 2*kv_dim] -> q_out, paged K/V.
__global__ void kv_append_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ q_out,
                                 __nv_bfloat16* __restrict__ k_cache, __nv_bfloat16* __restrict__ v_cache,
                                 const int* __restrict__ slots, int q_dim, int kv_dim, float q_scale) {
  pdl_launch_dependents();
  pdl_wait();
  const int t = blockIdx.x;
  const int tot = q_dim + 2 * kv_dim;
  const int slot = slots[t];
  for (int i = threadIdx.x; i < tot; i += blockDim.x) {
    const __nv_bfloat16 v = qkv[static_cast<size_t>(t) * tot + i];
    if (i < q_dim) q_out[static_cast<size_t>(t) * q_dim + i] = __float2bfloat16_rn(__bfloat162float(v) * q_scale);
    else if (slot >= 0) {
      if (i < q_dim + kv_dim) k_cache[static_cast<size_t>(slot) * kv_dim + (i - q_dim)] = v;
      else v_cache[static_cast<size_t>(slot) * kv_dim + (i - q_dim - kv_dim)] = v;
    }
  }
}

// y = a + b (residual add for unfused paths), 128-bit
__global__ void add_kernel(const __nv_bfloat16* __restrict__ a, const __nv_bfloat16* __restrict__ b,
                           __nv_bfloat16* __restrict__ out, size_t n8) {
  pdl_launch_dependents();
  pdl_wait();
  size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  if (i >= n8) return;
  uint4 x = reinterpret_cast<const uint4*>(a)[i], y = reinterpret_cast<const uint4*>(b)[i], o;
  const __nv_bfloat162* px = reinterpret_cast<const __nv_bfloat162*>(&x);
  const __nv_bfloat162* py = reinterpret_cast<const __nv_bfloat162*>(&y);
  __nv_bfloat162* po = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float2 f = __bfloat1622float2(px[j]), g = __bfloat1622float2(py[j]);
    po[j] = __floats2bfloat162_rn(f.x + g.x, f.y + g.y);
  }
  reinterpret_cast<uint4*>(out)[i] = o;
}

// Per-token dynamic fp8 (e4m3) quantisation of a GEMM input: q = x / s, s = amax / 448.
// scale_out[t] = s (x optional 1/rms of the row, so a following fp8 GEMM with gamma folded into
// its weights performs the whole RMSNorm + projection).  One CTA per token.
__global__ void quant_fp8_rows_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q,
                                      float* __restrict__ scale_out, int h, float eps, int with_rms) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float sh[32];
  const int t = blockIdx.x;
  const uint4* row = reinterpret_cast<const uint4*>(x + static_cast<size_t>(t) * h);
  float amax = 0.f, ss = 0.f;
  for (int i = threadIdx.x; i < h / 8; i += blockDim.x) {
    uint4 v = row[i];
    const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 f = __bfloat1622float2(p[j]);
      amax = fmaxf(amax, fmaxf(fabsf(f.x), fabsf(f.y)));
      ss += f.x * f.x + f.y * f.y;
    }
  }
  // block max via the sum helper on a monotone transform is awkward: do an explicit max reduce
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31, nw = (blockDim.x + 31) >> 5;
  if (l == 0) sh[w] = amax;
  __syncthreads();
  float m = (threadIdx.x < nw) ? sh[threadIdx.x] : 0.f;
  if (w == 0) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (l == 0) sh[0] = m;
  }
  __syncthreads();
  amax = sh[0];
  __syncthreads();
  ss = block_sum(ss, sh);
  const float s = amax > 0.f ? amax / 448.f : 1.f;
  const float inv = 1.f / s;
  if (threadIdx.x == 0) scale_out[t] = with_rms ? s * rsqrtf(ss / h + eps) : s;
  uint2* qrow = reinterpret_cast<uint2*>(q + static_cast<size_t>(t) * h);
  for (int i = threadIdx.x; i < h / 8; i += blockDim.x) {
    uint4 v = row[i];
    const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&v);
    uint8_t o[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float2 f = __bfloat1622float2(p[j]);
      o[2 * j] = __nv_cvt_float_to_fp8(f.x * inv, __NV_SATFINITE, __NV_E4M3);
      o[2 * j + 1] = __nv_cvt_float_to_fp8(f.y * inv, __NV_SATFINITE, __NV_E4M3);
    }
    qrow[i] = *reinterpret_cast<uint2*>(o);
  }
}

// MX (block-scaled) e4m3 quantisation of GEMM activations: one UE8M0 scale (2^e) per 32 consecutive K
// elements, q = x * rstd * 2^-e.  Scale bytes are written directly in the 512-byte chunk layout that
// GEMM expects for a token tile of `bn` rows (see GemmParams::sfb).  One CTA per token; a warp
// iteration covers 128 K elements (8 lanes x 4 elements = one 32-element block).  Padding rows of the last
// tile get scale 2^0 (a 0xFF byte would be NaN).
// with_rms: 0 = plain, 1 = 1/rms folded into the values before quantisation, 2 = values quantised as they are and the
// row's sum of squares written to sumsq_out (the consuming GEMM applies 1/rms in its epilogue: same numerics as the
// quantisation fused into a producing GEMM epilogue, csrc/gemm_tc.cu emit_q)
__global__ void quant_mxfp8_rows_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ q,
                                        uint8_t* __restrict__ sf, int tokens, int h, int bn, float eps, int with_rms,
                                        float* __restrict__ sumsq_out) {
  pdl_launch_dependents();
  pdl_wait();
  __shared__ float sh[32];
  const int t = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  const int nkc = h / 128;
  const int chunk_bytes = bn > 128 ? 1024 : 512;
  const int tile = t / bn, n = t % bn, r = n & 127;
  uint8_t* sfrow = sf + static_cast<size_t>(tile) * nkc * chunk_bytes + (n >> 7) * 512 + (r & 31) * 16 + (r >> 5) * 4;
  if (t >= tokens) {
    for (int i = threadIdx.x; i < nkc * 4; i += blockDim.x) sfrow[static_cast<size_t>(i >> 2) * chunk_bytes + (i & 3)] = 127;
    return;
  }
  const uint2* row = reinterpret_cast<const uint2*>(x + static_cast<size_t>(t) * h);
  float rs = 1.f;
  if (with_rms) {
    float ss = 0.f;
    for (int i = threadIdx.x; i < h / 4; i += blockDim.x) {
      const uint2 v = row[i];
      const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&v);
      const float2 a = __bfloat1622float2(p[0]), b = __bfloat1622float2(p[1]);
      ss += a.x * a.x + a.y * a.y + b.x * b.x + b.y * b.y;
    }
    ss = block_sum(ss, sh);
    if (with_rms == 2) {
      if (threadIdx.x == 0 && sumsq_out != nullptr) sumsq_out[t] = ss;
    } else {
      rs = rsqrtf(ss / h + eps);
    }
  }
  uint32_t* qrow = reinterpret_cast<uint32_t*>(q + static_cast<size_t>(t) * h);
  for (int kc = warp; kc < nkc; kc += nw) {
    const uint2 v = row[kc * 32 + lane];
    const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&v);
    const float2 a = __bfloat1622float2(p[0]), b = __bfloat1622float2(p[1]);
    const float f0 = a.x * rs, f1 = a.y * rs, f2 = b.x * rs, f3 = b.y * rs;
    float amax = fmaxf(fmaxf(fabsf(f0), fabsf(f1)), fmaxf(fabsf(f2), fabsf(f3)));
#pragma unroll
    for (int o = 1; o < 8; o <<= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    // e = ceil(log2(amax / 448)) clamped to the UE8M0 range; 2^e >= amax / 448 so |q| <= 448
    const uint32_t u = __float_as_uint(amax * (1.f / 448.f));
    int e = static_cast<int>(u >> 23) - 127 + ((u & 0x7FFFFFu) ? 1 : 0);
    e = max(-126, min(127, e));
    const float inv = __uint_as_float(static_cast<uint32_t>(127 - e) << 23);      // 2^-e (e = 127 -> 2^-127 denormal -> 0; unreachable for bf16 inputs)
    uint8_t o8[4];
    o8[0] = __nv_cvt_float_to_fp8(f0 * inv, __NV_SATFINITE, __NV_E4M3);
    o8[1] = __nv_cvt_float_to_fp8(f1 * inv, __NV_SATFINITE, __NV_E4M3);
    o8[2] = __nv_cvt_float_to_fp8(f2 * inv, __NV_SATFINITE, __NV_E4M3);
    o8[3] = __nv_cvt_float_to_fp8(f3 * inv, __NV_SATFINITE, __NV_E4M3);
    qrow[kc * 32 + lane] = *reinterpret_cast<uint32_t*>(o8);
    if ((lane & 7) == 0) sfrow[static_cast<size_t>(kc) * chunk_bytes + (lane >> 3)] = static_cast<uint8_t>(e + 127);
  }
}

// Stand-alone handoff primitives (used by the unfused / cudaMemcpyPeer comparator path)
__global__ void flag_wait_kernel(const uint32_t* flag, const uint32_t* epoch, uint32_t delta) {
  pdl_launch_dependents();
  pdl_wait();
  wait_flag_ge(flag, *reinterpret_cast<const volatile uint32_t*>(epoch) + delta);
}
__global__ void flag_signal_kernel(uint32_t* flag, uint32_t* epoch, uint32_t* bump_epoch, uint32_t* ack_flag) {
  pdl_launch_dependents();
  pdl_wait();
  __threadfence_system();
  if (flag != nullptr) {
    const uint32_t e = *reinterpret_cast<volatile uint32_t*>(epoch) + 1;
    *reinterpret_cast<volatile uint32_t*>(epoch) = e;
    st_release_sys(flag, e);
  }
  if (bump_epoch != nullptr) {
    const uint32_t e = *reinterpret_cast<volatile uint32_t*>(bump_epoch) + 1;
    *reinterpret_cast<volatile uint32_t*>(bump_epoch) = e;
    if (ack_flag != nullptr) st_release_sys(ack_flag, e);
  }
}

// Device-side bookkeeping of a decode step (keeps CUDA-graph replays host-free):
// positions += 1, kv_len += 1, slot = page(pos) * 64 + pos % 64 for every active sequence.
__global__ void decode_advance_kernel(int* positions, int* kv_len, int* slots, const int* q_len,
                                      const int* block_table, int max_pages, int n) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (q_len[i] <= 0) { slots[i] = -1; return; }
  const int pos = positions[i] + 1;
  positions[i] = pos;
  kv_len[i] = pos + 1;
  const int pg = pos / 64;
  slots[i] = (pg < max_pages) ? block_table[static_cast<size_t>(i) * max_pages + pg] * 64 + (pos % 64) : -1;
}

// After a (graph-captured) prefill: install the decode state of the sequence in batch row *row.
// row_map[i] = batch row of chunk sequence i whose prompt is complete after this chunk (< 0: skip).
__global__ void set_decode_state_kernel(int* positions, int* kv_len, int* q_len, const int* row_map, const int* kvlen,
                                        int n_rows) {
  pdl_launch_dependents();
  pdl_wait();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_rows) return;
  const int b = row_map[i];
  if (b < 0) return;
  const int n = kvlen[i];
  positions[b] = n - 1;
  kv_len[b] = n;
  q_len[b] = 1;
}

// Token read-back for the scheduler: one launch waits for the producers (sampler flags of every micro-batch group,
// prefill-done flag; the flags and the history ring may live on rank 0 = peer memory for follower ranks) and gathers
// every sequence's new tokens straight into mapped pinned host memory -- no NCCL broadcast, no host barrier.
__global__ void fetch_window_kernel(const int* history, int hist_stride, const int* cursors, int width, int* out,
                                    const FlagWait* waits, int n_waits, int* status) {
  pdl_launch_dependents();
  pdl_wait();
  if (threadIdx.x == 0) {
    for (int i = 0; i < n_waits; ++i) wait_flag_ge(waits[i].flag, waits[i].target);
    if (blockIdx.x == 0 && status != nullptr) {
      volatile uint32_t* ab = g_abort_word;
      *status = (ab != nullptr && *ab != 0u) ? 1 : 0;        // mapped host word: did any bounded wait give up?
    }
  }
  __syncthreads();
  const int b = blockIdx.x;
  const int cur = cursors[b];
  for (int j = threadIdx.x; j < width; j += blockDim.x)
    out[static_cast<size_t>(b) * width + j] =
        *reinterpret_cast<const volatile int*>(history + static_cast<size_t>(b) * hist_stride + ((cur + j) % hist_stride));
}

// ------------------------------------------------------------------ launchers
int launch_set_decode_state(int* positions, int* kv_len, int* q_len, const int* row_map, const int* kvlen, int n,
                            cudaStream_t s) {
  launch_kernel(set_decode_state_kernel, dim3((n + 63) / 64), dim3(64), 0, s, 1, positions, kv_len, q_len, row_map, kvlen, n);
  return static_cast<int>(cudaGetLastError());
}
int launch_fetch_window(const int* history, int hist_stride, const int* cursors, int rows, int width, int* out,
                        const FlagWait* waits, int n_waits, int* status, cudaStream_t s) {
  if (rows <= 0 || width <= 0) return 0;
  launch_kernel(fetch_window_kernel, dim3(rows), dim3(64), 0, s, 1, history, hist_stride, cursors, width, out, waits, n_waits,
                status);
  return static_cast<int>(cudaGetLastError());
}
int launch_decode_advance(int* positions, int* kv_len, int* slots, const int* q_len, const int* block_table,
                          int max_pages, int n, cudaStream_t s) {
  launch_kernel(decode_advance_kernel, dim3((n + 127) / 128), dim3(128), 0, s, 1, positions, kv_len, slots, q_len, block_table, max_pages, n);
  return static_cast<int>(cudaGetLastError());
}
int launch_rmsnorm(const void* x, const void* gamma, const void* residual, void* out, float* rstd_out, int tokens,
                   int h, float eps, int gemma_plus_one, cudaStream_t s) {
  if (h % 8) return -2;
  const int threads = h >= 4096 ? 512 : 256;
  launch_kernel(rmsnorm_kernel, dim3(tokens), dim3(threads), 0, s, 1, static_cast<const __nv_bfloat16*>(x), static_cast<const __nv_bfloat16*>(gamma),
                                            static_cast<const __nv_bfloat16*>(residual), static_cast<__nv_bfloat16*>(out),
                                            rstd_out, h, eps, gemma_plus_one);
  return static_cast<int>(cudaGetLastError());
}
int launch_layernorm(const void* x, const void* gamma, const void* beta, void* out, int tokens, int h, float eps,
                     cudaStream_t s) {
  launch_kernel(layernorm_kernel, dim3(tokens), dim3(256), 0, s, 1, static_cast<const __nv_bfloat16*>(x), static_cast<const __nv_bfloat16*>(gamma),
                                          static_cast<const __nv_bfloat16*>(beta), static_cast<__nv_bfloat16*>(out), h, eps);
  return static_cast<int>(cudaGetLastError());
}
int launch_embed(const int* ids, const void* table, const void* pos_table, const int* positions, void* out, int tokens,
                 int h, int vocab, float scale, const uint32_t* tok_flag, const uint32_t* tok_epoch, const uint32_t* pf_flag,
                 const uint32_t* pf_need, cudaStream_t s) {
  if (h % 8) return -2;
  launch_kernel(embed_kernel, dim3(tokens), dim3(256), 0, s, 1, ids, static_cast<const __nv_bfloat16*>(table),
                                      static_cast<const __nv_bfloat16*>(pos_table), positions,
                                      static_cast<__nv_bfloat16*>(out), h, vocab, scale, tok_flag, tok_epoch, pf_flag, pf_need);
  return static_cast<int>(cudaGetLastError());
}
int launch_kv_append(const void* qkv, void* q_out, void* k_cache, void* v_cache, const int* slots, int tokens,
                     int q_dim, int kv_dim, float q_scale, cudaStream_t s) {
  launch_kernel(kv_append_kernel, dim3(tokens), dim3(256), 0, s, 1, static_cast<const __nv_bfloat16*>(qkv), static_cast<__nv_bfloat16*>(q_out),
                                          static_cast<__nv_bfloat16*>(k_cache), static_cast<__nv_bfloat16*>(v_cache),
                                          slots, q_dim, kv_dim, q_scale);
  return static_cast<int>(cudaGetLastError());
}
int launch_add(const void* a, const void* b, void* out, size_t n, cudaStream_t s) {
  if (n % 8) return -2;
  const size_t n8 = n / 8;
  launch_kernel(add_kernel, dim3(static_cast<unsigned>((n8 + 255) / 256)), dim3(256), 0, s, 1, static_cast<const __nv_bfloat16*>(a),
                                                                      static_cast<const __nv_bfloat16*>(b),
                                                                      static_cast<__nv_bfloat16*>(out), n8);
  return static_cast<int>(cudaGetLastError());
}
int launch_quant_fp8_rows(const void* x, void* q, float* scale_out, int tokens, int h, float eps, int with_rms,
                          cudaStream_t s) {
  if (h % 8) return -2;
  launch_kernel(quant_fp8_rows_kernel, dim3(tokens), dim3(h >= 4096 ? 512 : 256), 0, s, 1,
                static_cast<const __nv_bfloat16*>(x), static_cast<uint8_t*>(q), scale_out, h, eps, with_rms);
  return static_cast<int>(cudaGetLastError());
}
int launch_quant_mxfp8_rows(const void* x, void* q, void* sf, int tokens, int h, int bn, float eps, int with_rms,
                            float* sumsq_out, cudaStream_t s) {
  if (h % 128 || bn < 32 || (bn & (bn - 1))) return -2;
  const int padded = (tokens + bn - 1) / bn * bn;
  launch_kernel(quant_mxfp8_rows_kernel, dim3(padded), dim3(h >= 4096 ? 512 : 256), 0, s, 1,
                static_cast<const __nv_bfloat16*>(x), static_cast<uint8_t*>(q), static_cast<uint8_t*>(sf), tokens, h, bn, eps,
                with_rms, sumsq_out);
  return static_cast<int>(cudaGetLastError());
}
int launch_flag_wait(const uint32_t* flag, const uint32_t* epoch, uint32_t delta, cudaStream_t s) {
  launch_kernel(flag_wait_kernel, dim3(1), dim3(1), 0, s, 1, flag, epoch, delta);
  return static_cast<int>(cudaGetLastError());
}
int launch_flag_signal(uint32_t* flag, uint32_t* epoch, uint32_t* bump_epoch, uint32_t* ack_flag, cudaStream_t s) {
  launch_kernel(flag_signal_kernel, dim3(1), dim3(1), 0, s, 1, flag, epoch, bump_epoch, ack_flag);
  return static_cast<int>(cudaGetLastError());
}

int set_wait_policy_elementwise(uint32_t* abort_word, unsigned long long limit_ns) {
  cudaError_t e = cudaMemcpyToSymbol(g_abort_word, &abort_word, sizeof(abort_word));
  if (e == cudaSuccess) e = cudaMemcpyToSymbol(g_wait_limit_ns, &limit_ns, sizeof(limit_ns));
  return static_cast<int>(e);
}

}  // namespace b2b
