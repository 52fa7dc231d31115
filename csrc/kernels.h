// C launcher API of the hand-written sm_90a kernels (no torch dependency: every .cu
// compiles in seconds with plain nvcc; csrc/binding.cpp is the only torch-facing file).
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace b2b {

// elementwise.cu
int launch_rmsnorm(const void* x, const void* gamma, const void* residual, void* out, float* rstd_out, int tokens,
                   int h, float eps, int gemma_plus_one, cudaStream_t s);
int launch_layernorm(const void* x, const void* gamma, const void* beta, void* out, int tokens, int h, float eps,
                     cudaStream_t s);
int launch_embed(const int* ids, const void* table, const void* pos_table, const int* positions, void* out, int tokens,
                 int h, int vocab, float scale, const uint32_t* tok_flag, const uint32_t* tok_epoch, const uint32_t* pf_flag,
                 const uint32_t* pf_need, cudaStream_t s);
int launch_kv_append(const void* qkv, void* q_out, void* k_cache, void* v_cache, const int* slots, int tokens,
                     int q_dim, int kv_dim, float q_scale, cudaStream_t s);
int launch_add(const void* a, const void* b, void* out, size_t n, cudaStream_t s);
int launch_quant_fp8_rows(const void* x, void* q, float* scale_out, int tokens, int h, float eps, int with_rms,
                          cudaStream_t s);
int launch_quant_mxfp8_rows(const void* x, void* q, void* sf, int tokens, int h, int bn, float eps, int with_rms,
                            float* sumsq_out, cudaStream_t s);
int launch_flag_wait(const uint32_t* flag, const uint32_t* epoch, uint32_t delta, cudaStream_t s);
int launch_decode_advance(int* positions, int* kv_len, int* slots, const int* q_len, const int* block_table,
                          int max_pages, int n, cudaStream_t s);
int launch_flag_signal(uint32_t* flag, uint32_t* epoch, uint32_t* bump_epoch, uint32_t* ack_flag, cudaStream_t s);

// attention.cu
int launch_attention(const void* q, const void* k_cache, const void* v_cache, void* out, const int* block_table,
                     const int* q_start, const int* q_len, const int* kv_len, float* ws, int seqs, int max_q,
                     int max_pages, int n_q, int n_kv, int head_dim, int window, float softcap, int splits,
                     cudaStream_t s);
int attn_rows(int G, int QB);
// attention_tc.cu: wgmma flash-attention forward for prefill chunks
bool attention_tc_supported(int n_q, int n_kv, int head_dim);
int launch_attention_tc(const void* q, const void* k_cache, const void* v_cache, void* out, const int* block_table,
                        const int* q_start, const int* q_len, const int* kv_len, int seqs, int max_q, int max_pages,
                        int n_tokens, int n_pages, int n_q, int n_kv, int head_dim, int window, float softcap,
                        int splits, float* ws, void* q_out8, void* q_sf, int q_bn, cudaStream_t s);
// merge pass of split-KV decode (shared by the CUDA-core and the tensor-core kernels)
int launch_attention_merge(void* out, const int* q_start, const int* q_len, const float* ws, int seqs, int n_q, int n_kv,
                           int head_dim, int splits, cudaStream_t s);
int attention_init();

// sampler.cu
int launch_sample(const float* logits, uint32_t* seen, int* out_tokens, int* peer_tokens, int* history,
                  const int* hist_pos, int* hist_pos_out, int hist_stride, int batch, int vocab, int ld, float softcap,
                  const float* temperature, const float* top_p, const float* rep_penalty, const uint32_t* seeds,
                  const uint32_t* step, uint32_t* signal_flag, uint32_t* signal_epoch, uint32_t* done_counter,
                  const int* row_map, cudaStream_t s);
// CTAs per sequence (1, 2, 4 or 8) that launch_sample runs a batch at on a device with `sms` SMs; 0 = the vocabulary
// does not fit in shared memory at any cluster size
int sample_cluster_size(int batch, int vocab, int sms);
int launch_set_decode_state(int* positions, int* kv_len, int* q_len, const int* row_map, const int* kvlen, int n,
                            cudaStream_t s);
// token-window read-back: wait for up to `n_waits` (flag, target) pairs, then out[b, j] = history[b, (cursor[b] + j) % stride]
struct FlagWait { const uint32_t* flag; uint32_t target; uint32_t pad; };
int launch_fetch_window(const int* history, int hist_stride, const int* cursors, int rows, int width, int* out,
                        const FlagWait* waits, int n_waits, int* status, cudaStream_t s);
int launch_mark_seen(const int* ids, const int* seq_of, uint32_t* seen, int n, int vocab, cudaStream_t s);

// bounded handoff waits: device abort word + time limit for the waits of each translation unit (0 / null = trap policy)
int set_wait_policy_gemm(uint32_t* abort_word, unsigned long long limit_ns);
int set_wait_policy_elementwise(uint32_t* abort_word, unsigned long long limit_ns);

// gemm_tc.cu
int gemm_tc_max_splitk(int bn, int epi, int stages);
int gemm_tc_init();

}  // namespace b2b
