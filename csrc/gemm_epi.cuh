// Fused GEMM epilogue math shared by the tensor-core kernels: applied to 16 consecutive token
// columns of one output feature after the accumulators have been read.
#pragma once
#include "common.cuh"
#include "gemm_tc.cuh"

namespace b2b {

__device__ __forceinline__ float epi_gelu_tanh(float x) {
  const float k0 = 0.7978845608028654f, k1 = 0.044715f;
  return 0.5f * x * (1.f + tanhf(k0 * (x + k1 * x * x * x)));
}
__device__ __forceinline__ float epi_silu(float x) { return x / (1.f + __expf(-x)); }

struct EpiCtx {
  int n_glob;        // output feature (row of W) owned by this thread
  int sect;          // QKV: 0 = q, 1 = k, 2 = v
  int f_in_sect;
  int q_dim, kv_dim;
  float inv_freq;
  float bias_v, wsc, wsc_up;
};

template <int EPI, bool FP8>
__device__ __forceinline__ EpiCtx epi_setup(const GemmParams& p, int tile_n, int row) {
  EpiCtx c;
  c.n_glob = tile_n * 128 + row;
  c.bias_v = (p.bias != nullptr) ? p.bias[c.n_glob] : 0.f;
  c.wsc = (FP8 && p.w_scale != nullptr) ? p.w_scale[c.n_glob] : 1.f;
  c.wsc_up = (FP8 && EPI == EPI_GLU && p.w_scale != nullptr && row < 64) ? p.w_scale[c.n_glob + 64] : 1.f;
  c.sect = 0; c.f_in_sect = 0; c.inv_freq = 0.f;
  c.q_dim = p.n_q_heads * p.head_dim;
  c.kv_dim = p.n_kv_heads * p.head_dim;
  if constexpr (EPI == EPI_QKV_ROPE) {
    const int f = c.n_glob;
    c.sect = (f < c.q_dim) ? 0 : (f < c.q_dim + c.kv_dim ? 1 : 2);
    c.f_in_sect = f - (c.sect == 0 ? 0 : (c.sect == 1 ? c.q_dim : c.q_dim + c.kv_dim));
    if (c.sect < 2 && p.rope_theta > 0.f) {
      const int j = (c.f_in_sect % p.head_dim) >> 1;   // rotary pair index (rows are pair-interleaved)
      c.inv_freq = exp2f(-(2.f * j / static_cast<float>(p.head_dim)) * log2f(p.rope_theta));
    }
  }
  return c;
}

// v[16]: accumulators of token columns c0 .. c0+15 (already reduced over split-K partials).
// xch: GLU exchange buffer [BN][64] holding the "up" half; rstd_s: per-token input scale.
template <int EPI, bool FP8>
__device__ __forceinline__ void epi_apply16(const GemmParams& p, const EpiCtx& e, const float* v, int c0, int tok0,
                                            int tile_n, int row, int lane, const float* rstd_s, const float* xch) {
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const int tok = tok0 + c0 + i;
    if (tok >= p.m_tok) continue;            // warp-uniform: padded token columns do no work
    const float rs = rstd_s[c0 + i];
    const float a = v[i] * rs * e.wsc + e.bias_v;
    if constexpr (EPI == EPI_PLAIN) {
      if (p.out_fp32) reinterpret_cast<float*>(p.out)[static_cast<size_t>(tok) * p.ld_out + e.n_glob] = a;
      else reinterpret_cast<__nv_bfloat16*>(p.out)[static_cast<size_t>(tok) * p.ld_out + e.n_glob] = __float2bfloat16_rn(a);
    } else if constexpr (EPI == EPI_GELU) {
      reinterpret_cast<__nv_bfloat16*>(p.out)[static_cast<size_t>(tok) * p.ld_out + e.n_glob] =
          __float2bfloat16_rn(epi_gelu_tanh(a));
    } else if constexpr (EPI == EPI_RESIDUAL) {
      const float r = __bfloat162float(p.residual[static_cast<size_t>(tok) * p.ld_res + e.n_glob]);
      reinterpret_cast<__nv_bfloat16*>(p.out)[static_cast<size_t>(tok) * p.ld_out + e.n_glob] = __float2bfloat16_rn(a + r);
    } else if constexpr (EPI == EPI_GLU) {
      const float u = xch[(c0 + i) * 64 + row] * rs * e.wsc_up;
      const float g = p.act_gelu ? epi_gelu_tanh(a) : epi_silu(a);
      reinterpret_cast<__nv_bfloat16*>(p.out)[static_cast<size_t>(tok) * p.ld_out + tile_n * 64 + row] =
          __float2bfloat16_rn(g * u);
    } else {   // EPI_QKV_ROPE
      float o = a;
      if (e.sect < 2 && p.rope_theta > 0.f) {
        // lanes (2j, 2j+1) hold (x_j, x_{j+hd/2}) thanks to the offline row interleave
        const float partner = __shfl_xor_sync(0xffffffffu, a, 1);
        float sn, cs;
        sincosf(static_cast<float>(p.positions[tok]) * e.inv_freq, &sn, &cs);
        o = (lane & 1) ? (a * cs + partner * sn) : (a * cs - partner * sn);
      }
      if (e.sect == 0) {
        p.q_out[static_cast<size_t>(tok) * e.q_dim + e.f_in_sect] = __float2bfloat16_rn(o * p.q_scale);
      } else {
        const int slot = p.slots[tok];
        __nv_bfloat16* dst = (e.sect == 1 ? p.k_cache : p.v_cache);
        if (slot >= 0) dst[static_cast<size_t>(slot) * e.kv_dim + e.f_in_sect] = __float2bfloat16_rn(o);
      }
    }
  }
}

// Publishes one finished tile of a piece-tail GEMM: once all `total_tiles` tiles have been stored
// (possibly into the peer GPU), the last arriver releases the handoff flag / bumps the epochs.
__device__ __forceinline__ void epi_publish_tile(const GemmParams& p, uint32_t total_tiles) {
  const uint32_t prev = atomicAdd(p.done_counter, 1u);
  if (prev == total_tiles - 1) {
    __threadfence_system();
    *p.done_counter = 0;
    if (p.signal_flag != nullptr) {
      const uint32_t e = *reinterpret_cast<volatile uint32_t*>(p.signal_epoch) + 1;
      *reinterpret_cast<volatile uint32_t*>(p.signal_epoch) = e;
      st_release_sys(p.signal_flag, e);
    }
    if (p.bump_epoch != nullptr) {
      const uint32_t e = *reinterpret_cast<volatile uint32_t*>(p.bump_epoch) + 1;
      *reinterpret_cast<volatile uint32_t*>(p.bump_epoch) = e;
      if (p.ack_flag != nullptr) st_release_sys(p.ack_flag, e);
    }
  }
}

}  // namespace b2b
