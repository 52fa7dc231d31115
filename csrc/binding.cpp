// Python bindings (torch extension `bee2bee_b200._C`).  The only torch-facing translation
// unit: it validates tensors, picks the current CUDA stream and calls the C launchers.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "gemm_tc.cuh"
#include "kernels.h"
#include "launch.cuh"
#include "peer.h"

using at::Tensor;
using OptT = c10::optional<Tensor>;

namespace {

inline cudaStream_t cur_stream() { return at::cuda::getCurrentCUDAStream().stream(); }

inline void check(int err, const char* what) {
  if (err != 0) {
    const char* msg = err > 0 ? cudaGetErrorString(static_cast<cudaError_t>(err)) : "invalid argument";
    TORCH_CHECK(false, what, " failed: code ", err, " (", msg, ")");
  }
}
template <typename T>
inline T* ptr_or_null(const OptT& t) {
  return (t.has_value() && t->defined()) ? reinterpret_cast<T*>(t->data_ptr()) : nullptr;
}
template <typename T>
inline T* as_ptr(int64_t addr) { return reinterpret_cast<T*>(static_cast<uintptr_t>(addr)); }

void check_bf16(const Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kBFloat16 && t.is_contiguous(), name,
              " must be a contiguous CUDA bf16 tensor");
}

// ---------------------------------------------------------------------- GEMM
// out[t, n] = epi(X[t,:] . W[n,:]).  Handoff pointers are raw device addresses (0 = unused)
// because they may live in IPC-mapped peer memory.
void gemm(const Tensor& w, const Tensor& x, int64_t out_ptr, int64_t ld_out, int64_t epi, int64_t bn,
          int64_t splitk, int64_t residual_ptr, int64_t ld_res, const OptT& bias, const OptT& rstd,
          bool norm_from_x, double eps, bool act_gelu, bool out_fp32,
          // qkv epilogue
          const OptT& q_out, const OptT& k_cache, const OptT& v_cache, const OptT& positions, const OptT& slots,
          int64_t n_q_heads, int64_t n_kv_heads, int64_t head_dim, double rope_theta, double q_scale,
          // handoff
          int64_t wait_flag, int64_t wait_epoch, int64_t signal_flag, int64_t signal_epoch, int64_t done_counter,
          int64_t free_flag, int64_t bump_epoch, int64_t ack_flag, int64_t dbg, const OptT& w_scale,
          const OptT& sfa, const OptT& sfb, int64_t stages, int64_t free_lag, int64_t out2_ptr,
          // fused MX quantisation of the output / RMSNorm statistics (raw addresses, 0 = off)
          int64_t q_out8, int64_t q_sf, int64_t ld_q, int64_t q_bn, int64_t sumsq_out, int64_t zero_buf, int64_t sumsq,
          // scaled RoPE: [head_dim/2] fp32 inverse frequencies, or none
          const OptT& rope_freq) {
  const bool fp8 = w.scalar_type() == at::kFloat8_e4m3fn;
  if (fp8) {
    TORCH_CHECK(x.scalar_type() == at::kFloat8_e4m3fn && w.is_cuda() && x.is_cuda() && w.is_contiguous() &&
                x.is_contiguous(), "fp8 gemm: w and x must be contiguous CUDA float8_e4m3fn");
    const bool mx = sfa.has_value();
    TORCH_CHECK(mx == sfb.has_value(), "MX fp8 gemm needs both sfa and sfb");
    if (mx) {
      const int64_t nkc = w.size(1) / 128, chunk = bn > 128 ? 1024 : 512;
      TORCH_CHECK(w.size(1) % 128 == 0 && bn >= 32, "MX fp8 gemm: K must be a multiple of 128 and bn >= 32");
      TORCH_CHECK(sfa->scalar_type() == at::kByte && sfa->is_contiguous() && sfa->numel() >= (w.size(0) / 128) * nkc * 512,
                  "MX fp8 gemm: sfa too small");
      TORCH_CHECK(sfb->scalar_type() == at::kByte && sfb->is_contiguous() &&
                      sfb->numel() >= ((x.size(0) + bn - 1) / bn) * nkc * chunk, "MX fp8 gemm: sfb too small");
    } else {
      TORCH_CHECK(w_scale.has_value() && w_scale->scalar_type() == at::kFloat, "fp8 gemm needs per-row w_scale (fp32)");
    }
  } else {
    check_bf16(w, "w");
    check_bf16(x, "x");
  }
  TORCH_CHECK(w.dim() == 2 && x.dim() == 2 && w.size(1) == x.size(1), "gemm: shape mismatch");
  c10::cuda::CUDAGuard guard(w.device());
  b2b::GemmParams p{};
  p.m_tok = static_cast<int>(x.size(0));
  p.n_out = static_cast<int>(w.size(0));
  p.k = static_cast<int>(w.size(1));
  p.splitk = static_cast<int8_t>(splitk);
  p.epi = static_cast<int8_t>(epi);
  p.out_fp32 = out_fp32 ? 1 : 0;
  p.act_gelu = act_gelu ? 1 : 0;
  p.fp8 = fp8 ? 1 : 0;
  p.stages = static_cast<int8_t>(stages);
  p.w_scale = ptr_or_null<const float>(w_scale);
  p.sfa = fp8 ? ptr_or_null<const uint8_t>(sfa) : nullptr;
  p.sfb = fp8 ? ptr_or_null<const uint8_t>(sfb) : nullptr;
  p.out = as_ptr<void>(out_ptr);
  p.ld_out = static_cast<int>(ld_out);
  p.out2 = as_ptr<void>(out2_ptr);
  p.q_out8 = as_ptr<uint8_t>(q_out8);
  p.q_sf = as_ptr<uint8_t>(q_sf);
  p.ld_q = static_cast<int>(ld_q);
  p.q_bn = static_cast<int16_t>(q_bn > 0 ? q_bn : 32);
  p.sumsq_out = as_ptr<float>(sumsq_out);
  p.zero_buf = as_ptr<float>(zero_buf);
  p.sumsq = as_ptr<const float>(sumsq);
  TORCH_CHECK(!p.q_out8 || (p.q_sf && p.sfa && p.ld_q % 128 == 0 && (epi == b2b::EPI_RESIDUAL || epi == b2b::EPI_GLU)),
              "fused output quantisation: MX GEMMs with residual / GLU epilogues, scale-factor buffer, row stride multiple of 128");
  p.residual = as_ptr<const __nv_bfloat16>(residual_ptr);
  p.ld_res = static_cast<int>(ld_res);
  p.bias = ptr_or_null<const float>(bias);
  p.rstd = ptr_or_null<const float>(rstd);
  TORCH_CHECK(!(fp8 && norm_from_x), "fp8 gemm: pass the combined activation scale through rstd");
  p.norm_src = norm_from_x ? reinterpret_cast<const __nv_bfloat16*>(x.data_ptr()) : nullptr;
  p.eps = static_cast<float>(eps);
  p.q_out = ptr_or_null<__nv_bfloat16>(q_out);
  p.k_cache = ptr_or_null<__nv_bfloat16>(k_cache);
  p.v_cache = ptr_or_null<__nv_bfloat16>(v_cache);
  p.positions = ptr_or_null<const int>(positions);
  p.slots = ptr_or_null<const int>(slots);
  p.n_q_heads = static_cast<int16_t>(n_q_heads);
  p.n_kv_heads = static_cast<int16_t>(n_kv_heads);
  p.head_dim = static_cast<int16_t>(head_dim);
  p.rope_theta = static_cast<float>(rope_theta);
  p.rope_freq = ptr_or_null<const float>(rope_freq);
  p.q_scale = static_cast<float>(q_scale);
  p.wait_flag = as_ptr<const uint32_t>(wait_flag);
  p.wait_epoch = as_ptr<const uint32_t>(wait_epoch);
  p.signal_flag = as_ptr<uint32_t>(signal_flag);
  p.signal_epoch = as_ptr<uint32_t>(signal_epoch);
  p.done_counter = as_ptr<uint32_t>(done_counter);
  p.free_flag = as_ptr<const uint32_t>(free_flag);
  p.bump_epoch = as_ptr<uint32_t>(bump_epoch);
  p.ack_flag = as_ptr<uint32_t>(ack_flag);
  p.free_lag = static_cast<uint8_t>(free_lag);
  p.dbg = as_ptr<unsigned long long>(dbg);
  if (p.epi == b2b::EPI_QKV_ROPE) {
    TORCH_CHECK(p.q_out && p.k_cache && p.v_cache && p.slots, "qkv epilogue needs q_out/k_cache/v_cache/slots");
    TORCH_CHECK(p.rope_theta <= 0.f || p.positions, "rope needs positions");
    if (rope_freq.has_value()) {
      TORCH_CHECK(rope_freq->is_cuda() && rope_freq->scalar_type() == at::kFloat && rope_freq->is_contiguous() &&
                      rope_freq->numel() == head_dim / 2 && rope_freq->device() == w.device(),
                  "rope_freq must be a contiguous fp32 tensor of head_dim/2 = ", head_dim / 2,
                  " entries on the GEMM's device");
      TORCH_CHECK(p.rope_theta > 0.f, "rope_freq needs rope_theta > 0");
    }
    TORCH_CHECK((p.n_q_heads * p.head_dim) % 128 == 0 && (p.n_kv_heads * p.head_dim) % 128 == 0,
                "q/kv widths must be multiples of 128");
    TORCH_CHECK(p.n_out == (p.n_q_heads + 2 * p.n_kv_heads) * p.head_dim, "qkv rows mismatch");
  }
  if (p.epi == b2b::EPI_RESIDUAL) TORCH_CHECK(p.residual != nullptr, "residual epilogue needs residual");
  if (p.epi == b2b::EPI_GLU) TORCH_CHECK(p.out != nullptr || (p.q_out8 != nullptr && p.sfa != nullptr), "GLU epilogue needs an output");
  if (p.signal_flag || p.bump_epoch) TORCH_CHECK(p.done_counter != nullptr, "handoff needs done_counter");
  check(b2b::launch_gemm_tc(p, w.data_ptr(), x.data_ptr(), static_cast<int>(bn), cur_stream()), "gemm_tc");
}

// Bounded handoff waits (call once per device after peer_alloc'ing the abort word): limit_ms == 0 restores "trap".
void set_wait_policy(int64_t abort_word, double limit_ms) {
  const auto ns = static_cast<unsigned long long>(limit_ms * 1e6);
  check(b2b::set_wait_policy_gemm(as_ptr<uint32_t>(abort_word), ns), "set_wait_policy(gemm)");
  check(b2b::set_wait_policy_elementwise(as_ptr<uint32_t>(abort_word), ns), "set_wait_policy(elementwise)");
}

void set_pdl(bool on) { b2b::g_pdl_mode = on ? 1 : 0; }
bool get_pdl() { return b2b::pdl_enabled(); }

int64_t gemm_max_splitk(int64_t bn, int64_t epi, int64_t stages) {
  return b2b::gemm_tc_max_splitk(static_cast<int>(bn), static_cast<int>(epi), static_cast<int>(stages));
}

// (ring depth, cluster split-K) that `gemm` runs for these arguments; fp8: 0 = bf16, 1 = per-row fp8, 2 = MX fp8
std::tuple<int64_t, int64_t> gemm_resolve(int64_t bn, int64_t epi, int64_t k, int64_t fp8, int64_t stages,
                                          int64_t splitk) {
  int st = 0, sk = 0;
  check(b2b::gemm_tc_resolve(static_cast<int>(bn), static_cast<int>(epi), static_cast<int>(k), static_cast<int>(fp8),
                             static_cast<int>(stages), static_cast<int>(splitk), &st, &sk),
        "gemm_resolve");
  return {st, sk};
}

void init_kernels(int64_t device) {
  c10::cuda::CUDAGuard guard(static_cast<c10::DeviceIndex>(device));
  check(b2b::gemm_tc_init(), "gemm_tc_init");
  check(b2b::attention_init(), "attention_init");
}

// ----------------------------------------------------------------- elementwise
// The elementwise kernels index every operand by the row length of x: a bf16 operand of another size or dtype would be
// read or written out of bounds, so each is checked here.
void check_bf16_numel(const Tensor& t, int64_t numel, const char* name) {
  check_bf16(t, name);
  TORCH_CHECK(t.numel() == numel, name, " has ", t.numel(), " elements, expected ", numel);
}

void rmsnorm(const Tensor& x, const Tensor& gamma, const OptT& residual, const OptT& out, const OptT& rstd_out,
             double eps, bool gemma_plus_one) {
  check_bf16(x, "x");
  TORCH_CHECK(x.dim() >= 1 && x.size(-1) > 0, "rmsnorm: x must have a nonempty last dimension");
  c10::cuda::CUDAGuard guard(x.device());
  const int h = static_cast<int>(x.size(-1));
  const int tokens = static_cast<int>(x.numel() / h);
  if (out.has_value() && out->defined()) {
    check_bf16_numel(gamma, h, "rmsnorm: gamma");
    check_bf16_numel(*out, x.numel(), "rmsnorm: out");
    if (residual.has_value() && residual->defined()) check_bf16_numel(*residual, x.numel(), "rmsnorm: residual");
  }
  if (rstd_out.has_value() && rstd_out->defined())
    TORCH_CHECK(rstd_out->is_cuda() && rstd_out->scalar_type() == at::kFloat && rstd_out->is_contiguous() &&
                    rstd_out->numel() >= tokens, "rmsnorm: rstd_out must be a contiguous CUDA fp32 tensor of >= ", tokens,
                " elements");
  check(b2b::launch_rmsnorm(x.data_ptr(), gamma.data_ptr(), ptr_or_null<void>(residual), ptr_or_null<void>(out),
                            ptr_or_null<float>(rstd_out), tokens, h, static_cast<float>(eps), gemma_plus_one ? 1 : 0,
                            cur_stream()),
        "rmsnorm");
}

void layernorm(const Tensor& x, const Tensor& gamma, const Tensor& beta, const Tensor& out, double eps) {
  check_bf16(x, "x");
  TORCH_CHECK(x.dim() >= 1 && x.size(-1) > 0, "layernorm: x must have a nonempty last dimension");
  c10::cuda::CUDAGuard guard(x.device());
  const int h = static_cast<int>(x.size(-1));
  check_bf16_numel(gamma, h, "layernorm: gamma");
  check_bf16_numel(beta, h, "layernorm: beta");
  check_bf16_numel(out, x.numel(), "layernorm: out");
  check(b2b::launch_layernorm(x.data_ptr(), gamma.data_ptr(), beta.data_ptr(), out.data_ptr(),
                              static_cast<int>(x.numel() / h), h, static_cast<float>(eps), cur_stream()),
        "layernorm");
}

void embed(int64_t ids_ptr, const Tensor& table, const OptT& pos_table, const OptT& positions, const Tensor& out,
           double scale, int64_t tok_flag, int64_t tok_epoch, int64_t pf_flag, int64_t pf_need) {
  check_bf16(table, "table");
  TORCH_CHECK(table.dim() == 2 && table.size(0) > 0 && table.size(1) > 0, "embed: table must be [vocab, h]");
  c10::cuda::CUDAGuard guard(table.device());
  const int h = static_cast<int>(table.size(1));
  check_bf16(out, "embed: out");
  TORCH_CHECK(out.numel() % h == 0, "embed: out has ", out.numel(), " elements, not a multiple of h = ", h);
  const bool has_pos = pos_table.has_value() && pos_table->defined();
  TORCH_CHECK(has_pos == (positions.has_value() && positions->defined()), "embed: pos_table and positions go together");
  if (has_pos) {
    check_bf16(*pos_table, "embed: pos_table");
    TORCH_CHECK(pos_table->dim() == 2 && pos_table->size(0) > 0 && pos_table->size(1) == h, "embed: pos_table must be [n_pos, ",
                h, "]");
    TORCH_CHECK(positions->is_cuda() && positions->scalar_type() == at::kInt && positions->is_contiguous() &&
                    positions->numel() >= out.numel() / h,
                "embed: positions must be contiguous CUDA int32 with one entry per token");
  }
  check(b2b::launch_embed(as_ptr<const int>(ids_ptr), table.data_ptr(), ptr_or_null<void>(pos_table),
                          ptr_or_null<const int>(positions), out.data_ptr(), static_cast<int>(out.numel() / h), h,
                          static_cast<int>(table.size(0)), static_cast<float>(scale), as_ptr<const uint32_t>(tok_flag),
                          as_ptr<const uint32_t>(tok_epoch), as_ptr<const uint32_t>(pf_flag), as_ptr<const uint32_t>(pf_need),
                          cur_stream()),
        "embed");
}

void kv_append(const Tensor& qkv, const Tensor& q_out, const Tensor& k_cache, const Tensor& v_cache,
               const Tensor& slots, int64_t q_dim, int64_t kv_dim, double q_scale) {
  check_bf16(qkv, "qkv");
  TORCH_CHECK(q_dim > 0 && kv_dim > 0 && qkv.dim() == 2 && qkv.size(1) == q_dim + 2 * kv_dim,
              "kv_append: qkv must be [T, q_dim + 2 * kv_dim] = [T, ", q_dim + 2 * kv_dim, "]");
  check_bf16(q_out, "kv_append: q_out");
  TORCH_CHECK(q_out.numel() >= qkv.size(0) * q_dim, "kv_append: q_out holds fewer than T rows of q_dim");
  check_bf16(k_cache, "kv_append: k_cache");
  check_bf16(v_cache, "kv_append: v_cache");
  TORCH_CHECK(k_cache.numel() % kv_dim == 0 && v_cache.numel() == k_cache.numel(),
              "kv_append: k_cache and v_cache must be equal-sized rows of kv_dim");
  TORCH_CHECK(slots.is_cuda() && slots.scalar_type() == at::kInt && slots.is_contiguous() && slots.numel() >= qkv.size(0),
              "kv_append: slots must be contiguous CUDA int32 with one entry per token");
  c10::cuda::CUDAGuard guard(qkv.device());
  check(b2b::launch_kv_append(qkv.data_ptr(), q_out.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(),
                              reinterpret_cast<const int*>(slots.data_ptr()), static_cast<int>(qkv.size(0)),
                              static_cast<int>(q_dim), static_cast<int>(kv_dim), static_cast<float>(q_scale),
                              cur_stream()),
        "kv_append");
}

void add(const Tensor& a, const Tensor& b, const Tensor& out) {
  check_bf16(a, "a");
  check_bf16_numel(b, a.numel(), "add: b");
  check_bf16_numel(out, a.numel(), "add: out");
  c10::cuda::CUDAGuard guard(a.device());
  check(b2b::launch_add(a.data_ptr(), b.data_ptr(), out.data_ptr(), static_cast<size_t>(a.numel()), cur_stream()),
        "add");
}

void quant_fp8_rows(const Tensor& x, const Tensor& q, const Tensor& scale_out, double eps, bool with_rms) {
  check_bf16(x, "x");
  TORCH_CHECK(q.scalar_type() == at::kFloat8_e4m3fn && q.is_contiguous() && scale_out.scalar_type() == at::kFloat,
              "quant_fp8_rows: q must be float8_e4m3fn, scale fp32");
  c10::cuda::CUDAGuard guard(x.device());
  const int h = static_cast<int>(x.size(-1));
  check(b2b::launch_quant_fp8_rows(x.data_ptr(), q.data_ptr(), reinterpret_cast<float*>(scale_out.data_ptr()),
                                   static_cast<int>(x.numel() / h), h, static_cast<float>(eps), with_rms ? 1 : 0,
                                   cur_stream()),
        "quant_fp8_rows");
}

void quant_mxfp8_rows(const Tensor& x, const Tensor& q, const Tensor& sf, int64_t bn, double eps, int64_t with_rms,
                      const OptT& sumsq_out) {
  check_bf16(x, "x");
  TORCH_CHECK(q.scalar_type() == at::kFloat8_e4m3fn && q.is_contiguous() && sf.scalar_type() == at::kByte &&
                  sf.is_contiguous(), "quant_mxfp8_rows: q must be float8_e4m3fn, sf uint8");
  c10::cuda::CUDAGuard guard(x.device());
  const int h = static_cast<int>(x.size(-1));
  const int tokens = static_cast<int>(x.numel() / h);
  TORCH_CHECK(sf.numel() >= ((tokens + bn - 1) / bn) * (h / 128) * (bn > 128 ? 1024 : 512), "quant_mxfp8_rows: sf too small");
  check(b2b::launch_quant_mxfp8_rows(x.data_ptr(), q.data_ptr(), sf.data_ptr(), tokens, h, static_cast<int>(bn),
                                     static_cast<float>(eps), static_cast<int>(with_rms), ptr_or_null<float>(sumsq_out),
                                     cur_stream()),
        "quant_mxfp8_rows");
}

void flag_wait(int64_t flag, int64_t epoch, int64_t delta) {
  check(b2b::launch_flag_wait(as_ptr<const uint32_t>(flag), as_ptr<const uint32_t>(epoch),
                              static_cast<uint32_t>(delta), cur_stream()),
        "flag_wait");
}
void decode_advance(const Tensor& positions, const Tensor& kv_len, const Tensor& slots, const Tensor& q_len,
                    const Tensor& block_table) {
  c10::cuda::CUDAGuard guard(positions.device());
  check(b2b::launch_decode_advance(reinterpret_cast<int*>(positions.data_ptr()), reinterpret_cast<int*>(kv_len.data_ptr()),
                                   reinterpret_cast<int*>(slots.data_ptr()),
                                   reinterpret_cast<const int*>(q_len.data_ptr()),
                                   reinterpret_cast<const int*>(block_table.data_ptr()),
                                   static_cast<int>(block_table.size(1)), static_cast<int>(positions.numel()),
                                   cur_stream()),
        "decode_advance");
}
void flag_signal(int64_t flag, int64_t epoch, int64_t bump_epoch, int64_t ack_flag) {
  check(b2b::launch_flag_signal(as_ptr<uint32_t>(flag), as_ptr<uint32_t>(epoch), as_ptr<uint32_t>(bump_epoch),
                                as_ptr<uint32_t>(ack_flag), cur_stream()),
        "flag_signal");
}

// -------------------------------------------------------------------- attention
// query-chunk length from which prefill chunks run on the tensor-core kernel (0 = never, decode included)
static int64_t g_attn_tc_min_q = 2;
void set_attn_tc_min_q(int64_t v) { g_attn_tc_min_q = v; }
int64_t get_attn_tc_min_q() { return g_attn_tc_min_q; }

// The attention kernel of a call.  use_tc: -1 = default: decode (max_q == 1, the GQA group stacked into the MMA rows)
// and prefill chunks of at least tc_min_q queries run on the tensor-core kernel; 1 = force the tensor-core kernel; 0 =
// force the CUDA-core kernel.  The tensor-core kernel also needs tc_min_q > 0 and a GQA layout it supports; every other
// call runs on the CUDA-core kernel.
bool attention_uses_tc(int64_t max_q, int64_t n_q, int64_t n_kv, int64_t head_dim, int64_t use_tc) {
  if (use_tc == 0 || g_attn_tc_min_q <= 0 ||
      !b2b::attention_tc_supported(static_cast<int>(n_q), static_cast<int>(n_kv), static_cast<int>(head_dim)))
    return false;
  return use_tc > 0 || max_q == 1 || max_q >= g_attn_tc_min_q;
}

void attention(const Tensor& q, const Tensor& k_cache, const Tensor& v_cache, const Tensor& out,
               const Tensor& block_table, const Tensor& q_start, const Tensor& q_len, const Tensor& kv_len,
               const OptT& ws, int64_t max_q, int64_t n_q, int64_t n_kv, int64_t head_dim, int64_t window,
               double softcap, int64_t splits, int64_t use_tc, int64_t fq_out, int64_t fq_sf, int64_t fq_bn) {
  check_bf16(q, "q");
  c10::cuda::CUDAGuard guard(q.device());
  TORCH_CHECK(block_table.scalar_type() == at::kInt && q_len.scalar_type() == at::kInt, "int32 metadata expected");
  const int seqs = static_cast<int>(q_len.size(0));
  const bool tc = attention_uses_tc(max_q, n_q, n_kv, head_dim, use_tc);
  // split-KV: the CUDA-core kernel, or the tensor-core kernel on decode (it runs prefill chunks unsplit)
  if (splits > 1 && (!tc || max_q == 1)) {
    TORCH_CHECK(ws.has_value(), "split-KV needs a workspace");
    const int64_t R = b2b::attn_rows(static_cast<int>(n_q / n_kv), 1);
    TORCH_CHECK(ws->numel() >= seqs * n_kv * splits * R * (head_dim + 2), "attention workspace too small");
  }
  if (tc) {
    check(b2b::launch_attention_tc(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), out.data_ptr(),
                                   reinterpret_cast<const int*>(block_table.data_ptr()),
                                   reinterpret_cast<const int*>(q_start.data_ptr()),
                                   reinterpret_cast<const int*>(q_len.data_ptr()),
                                   reinterpret_cast<const int*>(kv_len.data_ptr()), seqs, static_cast<int>(max_q),
                                   static_cast<int>(block_table.size(1)), static_cast<int>(q.size(0)),
                                   static_cast<int>(k_cache.size(0)), static_cast<int>(n_q), static_cast<int>(n_kv),
                                   static_cast<int>(head_dim), static_cast<int>(window), static_cast<float>(softcap),
                                   static_cast<int>(splits), ptr_or_null<float>(ws), as_ptr<void>(fq_out), as_ptr<void>(fq_sf),
                                   static_cast<int>(fq_bn), cur_stream()),
          "attention_tc");
    return;
  }
  TORCH_CHECK(fq_out == 0, "fused output quantisation needs the tensor-core attention kernel");
  check(b2b::launch_attention(q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), out.data_ptr(),
                              reinterpret_cast<const int*>(block_table.data_ptr()),
                              reinterpret_cast<const int*>(q_start.data_ptr()),
                              reinterpret_cast<const int*>(q_len.data_ptr()),
                              reinterpret_cast<const int*>(kv_len.data_ptr()), ptr_or_null<float>(ws), seqs,
                              static_cast<int>(max_q), static_cast<int>(block_table.size(1)), static_cast<int>(n_q),
                              static_cast<int>(n_kv), static_cast<int>(head_dim), static_cast<int>(window),
                              static_cast<float>(softcap), static_cast<int>(splits), cur_stream()),
        "attention");
}

// ---------------------------------------------------------------------- sampler
// bound keyword-only, with ops.sample's parameter names and no defaults: the optional per-row tensors share one type,
// so a positional slip would still pass every check and sample with the wrong control
void sample(const Tensor& logits, const Tensor& out_tokens, const OptT& seen, const OptT& temperature,
            const OptT& top_p, const OptT& rep_penalty, const OptT& seeds, const OptT& step, int64_t peer_tokens,
            int64_t history, const OptT& hist_pos, int64_t hist_stride, int64_t signal_flag, int64_t signal_epoch,
            int64_t done_counter, int64_t vocab, double softcap, int64_t row_map, const OptT& top_k,
            const OptT& min_p, const OptT& counts, const OptT& presence, const OptT& frequency,
            const OptT& bias_ids, const OptT& bias_vals, const OptT& bias_n) {
  TORCH_CHECK(logits.is_cuda() && logits.scalar_type() == at::kFloat && logits.stride(1) == 1, "logits: fp32");
  // top_k / min_p are per-sequence state like temperature: one entry per state row (logits row b reads row
  // row_map[b], or b without a row_map)
  const bool has_temp = temperature.has_value() && temperature->defined();
  const int64_t state_rows = has_temp ? temperature->numel() : logits.size(0);
  auto check_row_param = [&](const OptT& t, at::ScalarType dtype, const char* name) {
    if (!(t.has_value() && t->defined())) return;
    TORCH_CHECK(t->scalar_type() == dtype && t->device() == logits.device() && t->dim() == 1 && t->is_contiguous(),
                name, " must be a contiguous 1-D ", dtype == at::kInt ? "int32" : "float32",
                " tensor on the logits' device");
    TORCH_CHECK(t->numel() == state_rows && (row_map != 0 || t->numel() >= logits.size(0)), name, " has ", t->numel(),
                " entries; expected one per state row (", state_rows, ")");
  };
  check_row_param(top_k, at::kInt, "top_k");
  check_row_param(min_p, at::kFloat, "min_p");
  check_row_param(presence, at::kFloat, "presence");
  check_row_param(frequency, at::kFloat, "frequency");
  const int64_t V = vocab > 0 ? vocab : logits.size(1);
  const bool has_counts = counts.has_value() && counts->defined();
  if (has_counts) {
    // [state rows, cstride] int16, rows padded to a multiple of 8 ids so that 4 ids are one aligned 8-byte load
    const Tensor& c = *counts;
    TORCH_CHECK(c.scalar_type() == at::kShort && c.device() == logits.device() && c.dim() == 2 && c.stride(1) == 1,
                "counts must be a 2-D int16 tensor with unit column stride on the logits' device");
    TORCH_CHECK(c.size(0) == state_rows && (row_map != 0 || c.size(0) >= logits.size(0)), "counts has ", c.size(0),
                " rows; expected one per state row (", state_rows, ")");
    TORCH_CHECK(c.size(1) >= V && c.stride(0) >= V && c.stride(0) % 8 == 0 &&
                    (reinterpret_cast<uintptr_t>(c.data_ptr()) & 7) == 0,
                "counts rows must hold the vocabulary (", V, " ids) at a row stride that is a multiple of 8 ids, "
                "from an 8-byte aligned address; got ", c.size(1), " ids at stride ", c.stride(0));
  }
  // logit bias: [state rows, width] int32 ids and fp32 values, and the entries in use per row (bias_n, like top_k)
  const bool has_ids = bias_ids.has_value() && bias_ids->defined();
  const bool has_vals = bias_vals.has_value() && bias_vals->defined();
  const bool has_bias = bias_n.has_value() && bias_n->defined();
  TORCH_CHECK(has_ids == has_bias && has_vals == has_bias, "bias_ids, bias_vals and bias_n go together");
  if (has_bias) {
    check_row_param(bias_n, at::kInt, "bias_n");
    auto check_table = [&](const Tensor& t, at::ScalarType dtype, const char* name) {
      TORCH_CHECK(t.scalar_type() == dtype && t.device() == logits.device() && t.dim() == 2 && t.is_contiguous(),
                  name, " must be a contiguous 2-D ", dtype == at::kInt ? "int32" : "float32",
                  " tensor on the logits' device");
      TORCH_CHECK(t.size(0) == state_rows, name, " has ", t.size(0), " rows; expected one per state row (",
                  state_rows, ")");
    };
    check_table(*bias_ids, at::kInt, "bias_ids");
    check_table(*bias_vals, at::kFloat, "bias_vals");
    TORCH_CHECK(bias_ids->size(1) == bias_vals->size(1), "bias_ids and bias_vals must have the same width; got ",
                bias_ids->size(1), " and ", bias_vals->size(1));
  }
  c10::cuda::CUDAGuard guard(logits.device());
  b2b::SampleParams p{};
  p.logits = reinterpret_cast<const float*>(logits.data_ptr());
  p.seen = ptr_or_null<uint32_t>(seen);
  p.out_tokens = reinterpret_cast<int*>(out_tokens.data_ptr());
  p.peer_tokens = as_ptr<int>(peer_tokens);
  p.history = as_ptr<int>(history);
  p.hist_pos = p.hist_pos_out = ptr_or_null<int>(hist_pos);
  p.hist_stride = static_cast<int>(hist_stride);
  p.vocab = static_cast<int>(V);
  p.ld = static_cast<int>(logits.stride(0));
  p.softcap = static_cast<float>(softcap);
  p.temperature = ptr_or_null<const float>(temperature);
  p.top_p = ptr_or_null<const float>(top_p);
  p.top_k = ptr_or_null<const int>(top_k);
  p.min_p = ptr_or_null<const float>(min_p);
  p.rep_penalty = ptr_or_null<const float>(rep_penalty);
  p.counts = ptr_or_null<int16_t>(counts);
  p.cstride = has_counts ? static_cast<int>(counts->stride(0)) : 0;
  p.presence = ptr_or_null<const float>(presence);
  p.frequency = ptr_or_null<const float>(frequency);
  p.bias_ids = ptr_or_null<const int>(bias_ids);
  p.bias_vals = ptr_or_null<const float>(bias_vals);
  p.bias_n = ptr_or_null<const int>(bias_n);
  p.bias_stride = has_bias ? static_cast<int>(bias_ids->size(1)) : 0;
  p.seeds = ptr_or_null<const uint32_t>(seeds);
  p.step = ptr_or_null<const uint32_t>(step);
  p.signal_flag = as_ptr<uint32_t>(signal_flag);
  p.signal_epoch = as_ptr<uint32_t>(signal_epoch);
  p.done_counter = as_ptr<uint32_t>(done_counter);
  p.row_map = as_ptr<const int>(row_map);
  check(b2b::launch_sample(p, static_cast<int>(logits.size(0)), cur_stream()), "sample");
}

// CTAs per sequence that `sample` runs a batch of `batch` rows at on the current device (0 = vocabulary too large)
int64_t sample_cluster_size(int64_t batch, int64_t vocab) {
  int dev = 0, sms = 0;
  check(static_cast<int>(cudaGetDevice(&dev)), "cudaGetDevice");
  check(static_cast<int>(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev)), "cudaDeviceGetAttribute");
  return b2b::sample_cluster_size(static_cast<int>(batch), static_cast<int>(vocab), sms);
}

void set_decode_state(const Tensor& positions, const Tensor& kv_len, const Tensor& q_len, int64_t row_map, int64_t kvlen,
                      int64_t n) {
  c10::cuda::CUDAGuard guard(positions.device());
  check(b2b::launch_set_decode_state(reinterpret_cast<int*>(positions.data_ptr()), reinterpret_cast<int*>(kv_len.data_ptr()),
                                     reinterpret_cast<int*>(q_len.data_ptr()), as_ptr<const int>(row_map),
                                     as_ptr<const int>(kvlen), static_cast<int>(n), cur_stream()),
        "set_decode_state");
}

// history / cursors / out / waits are raw addresses: the ring may be peer memory, the rest mapped pinned host memory
void fetch_window(int64_t history, int64_t hist_stride, int64_t cursors, int64_t rows, int64_t width, int64_t out,
                  int64_t waits, int64_t n_waits, int64_t status) {
  check(b2b::launch_fetch_window(as_ptr<const int>(history), static_cast<int>(hist_stride), as_ptr<const int>(cursors),
                                 static_cast<int>(rows), static_cast<int>(width), as_ptr<int>(out),
                                 as_ptr<const b2b::FlagWait>(waits), static_cast<int>(n_waits), as_ptr<int>(status),
                                 cur_stream()),
        "fetch_window");
}

void mark_seen(const Tensor& ids, const Tensor& seq_of, const Tensor& seen, int64_t vocab) {
  c10::cuda::CUDAGuard guard(ids.device());
  check(b2b::launch_mark_seen(reinterpret_cast<const int*>(ids.data_ptr()),
                              reinterpret_cast<const int*>(seq_of.data_ptr()),
                              reinterpret_cast<uint32_t*>(seen.data_ptr()), static_cast<int>(ids.numel()),
                              static_cast<int>(vocab), cur_stream()),
        "mark_seen");
}

// ------------------------------------------------------------------ peer memory
int64_t peer_alloc(int64_t bytes) {
  void* p = nullptr;
  check(b2b::peer_alloc(static_cast<size_t>(bytes), &p), "peer_alloc");
  return static_cast<int64_t>(reinterpret_cast<uintptr_t>(p));
}
void peer_free(int64_t p) { check(b2b::peer_free(as_ptr<void>(p)), "peer_free"); }
py::bytes ipc_export(int64_t p) {
  char h[64];
  check(b2b::ipc_export(as_ptr<void>(p), h), "cudaIpcGetMemHandle");
  return py::bytes(h, 64);
}
int64_t ipc_import(const std::string& handle) {
  TORCH_CHECK(handle.size() == 64, "IPC handle must be 64 bytes");
  void* p = nullptr;
  check(b2b::ipc_import(handle.data(), &p), "cudaIpcOpenMemHandle");
  return static_cast<int64_t>(reinterpret_cast<uintptr_t>(p));
}
void ipc_close(int64_t p) { check(b2b::ipc_close(as_ptr<void>(p)), "cudaIpcCloseMemHandle"); }
void enable_peer_access(int64_t dev, int64_t peer) {
  check(b2b::enable_peer_access(static_cast<int>(dev), static_cast<int>(peer)), "cudaDeviceEnablePeerAccess");
}
bool can_access_peer(int64_t dev, int64_t peer) {
  return b2b::can_access_peer(static_cast<int>(dev), static_cast<int>(peer)) != 0;
}
void memcpy_peer(int64_t dst, int64_t dst_dev, int64_t src, int64_t src_dev, int64_t bytes) {
  check(b2b::memcpy_peer_async(as_ptr<void>(dst), static_cast<int>(dst_dev), as_ptr<const void>(src),
                               static_cast<int>(src_dev), static_cast<size_t>(bytes), cur_stream()),
        "cudaMemcpyPeerAsync");
}
std::pair<int64_t, int64_t> host_ring_alloc(int64_t bytes) {
  void *h = nullptr, *d = nullptr;
  check(b2b::host_ring_alloc(static_cast<size_t>(bytes), &h, &d), "cudaHostAlloc");
  return {static_cast<int64_t>(reinterpret_cast<uintptr_t>(h)), static_cast<int64_t>(reinterpret_cast<uintptr_t>(d))};
}
void host_ring_free(int64_t h) { check(b2b::host_ring_free(as_ptr<void>(h)), "cudaFreeHost"); }

// View raw (possibly peer-mapped or host-mapped) memory as a tensor; no ownership.
Tensor tensor_from_ptr(int64_t p, std::vector<int64_t> sizes, const std::string& dtype, int64_t device) {
  at::ScalarType st = dtype == "bf16" ? at::kBFloat16 : dtype == "f32" ? at::kFloat : dtype == "i32" ? at::kInt
                      : dtype == "u8" ? at::kByte : at::kLong;
  auto opts = at::TensorOptions().dtype(st);
  opts = device >= 0 ? opts.device(at::kCUDA, static_cast<c10::DeviceIndex>(device)) : opts.device(at::kCPU);
  return at::from_blob(as_ptr<void>(p), sizes, opts);
}

}  // namespace

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "bee2bee_b200 native sm_90a kernels + NVLink peer-memory runtime";
  m.def("gemm", &gemm);
  m.def("gemm_max_splitk", &gemm_max_splitk);
  m.def("gemm_resolve", &gemm_resolve, py::arg("bn"), py::arg("epi"), py::arg("k"), py::arg("fp8"), py::arg("stages"),
        py::arg("splitk"));
  m.def("init_kernels", &init_kernels);
  m.def("set_pdl", &set_pdl);
  m.def("get_pdl", &get_pdl);
  m.def("rmsnorm", &rmsnorm);
  m.def("layernorm", &layernorm);
  m.def("embed", &embed);
  m.def("kv_append", &kv_append);
  m.def("add", &add);
  m.def("quant_fp8_rows", &quant_fp8_rows);
  m.def("quant_mxfp8_rows", &quant_mxfp8_rows);
  m.def("flag_wait", &flag_wait);
  m.def("flag_signal", &flag_signal);
  m.def("decode_advance", &decode_advance);
  m.def("attention", &attention);
  m.def("attention_uses_tc", &attention_uses_tc, py::arg("max_q"), py::arg("n_q"), py::arg("n_kv"), py::arg("head_dim"),
        py::arg("use_tc") = -1);
  m.def("set_attn_tc_min_q", &set_attn_tc_min_q);
  m.def("get_attn_tc_min_q", &get_attn_tc_min_q);
  m.def("sample", &sample, py::kw_only(), py::arg("logits"), py::arg("out_tokens"), py::arg("seen"),
        py::arg("temperature"), py::arg("top_p"), py::arg("rep_penalty"), py::arg("seeds"), py::arg("step"),
        py::arg("peer_tokens"), py::arg("history"), py::arg("hist_pos"), py::arg("hist_stride"),
        py::arg("signal_flag"), py::arg("signal_epoch"), py::arg("done_counter"), py::arg("vocab"), py::arg("softcap"),
        py::arg("row_map"), py::arg("top_k"), py::arg("min_p"), py::arg("counts"), py::arg("presence"),
        py::arg("frequency"), py::arg("bias_ids"), py::arg("bias_vals"), py::arg("bias_n"));
  m.def("sample_cluster_size", &sample_cluster_size, py::arg("batch"), py::arg("vocab"));
  m.def("mark_seen", &mark_seen);
  m.def("set_decode_state", &set_decode_state);
  m.def("fetch_window", &fetch_window);
  m.def("set_wait_policy", &set_wait_policy);
  m.def("peer_alloc", &peer_alloc);
  m.def("peer_free", &peer_free);
  m.def("ipc_export", &ipc_export);
  m.def("ipc_import", &ipc_import);
  m.def("ipc_close", &ipc_close);
  m.def("enable_peer_access", &enable_peer_access);
  m.def("can_access_peer", &can_access_peer);
  m.def("memcpy_peer", &memcpy_peer);
  m.def("host_ring_alloc", &host_ring_alloc);
  m.def("host_ring_free", &host_ring_free);
  m.def("tensor_from_ptr", &tensor_from_ptr);
}
