// Host launch API of the sm_90a kernels (entry points and file names keep the names they were introduced with). Plain C types only: bindings.cpp adapts at::Tensor to these.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200 {

// last error raised by a launcher on this thread ("" if none); cleared by take_last_error()
const char* take_last_error();

// ---- norm.cu --------------------------------------------------------------------------------------------------
// y = x * rsqrt(mean(x^2) + eps) * w (+ b) ; optional fused residual: h = x + residual (h written to res_out)
void rms_norm_fwd(const void* x, const void* residual, const void* w, const void* b, void* y, void* res_out,
                  float* rstd, int64_t rows, int cols, float eps, int dtype, cudaStream_t s);
void rms_norm_bwd(const void* dy, const void* x, const void* w, const float* rstd, void* dx, float* dw_partial,
                  float* db_partial, int64_t rows, int cols, int dtype, int n_partial, cudaStream_t s);
void layer_norm_fwd(const void* x, const void* w, const void* b, void* y, float* mean, float* rstd, int64_t rows,
                    int cols, float eps, int dtype, cudaStream_t s);
void layer_norm_bwd(const void* dy, const void* x, const void* w, const float* mean, const float* rstd, void* dx,
                    float* dw_partial, float* db_partial, int64_t rows, int cols, int dtype, int n_partial,
                    cudaStream_t s);
// out[c] = sum_p partial[p, c]  (fp32 in, `dtype` out)
void reduce_partials(const float* partial, void* out, int n_partial, int cols, int dtype, cudaStream_t s);
int norm_bwd_num_partials(int64_t rows);

// ---- elementwise.cu -------------------------------------------------------------------------------------------
// out = silu(gate) * up. If up == nullptr, x is [rows, 2*cols] packed (gate | up).
void swiglu_fwd(const void* gate, const void* up, void* out, int64_t rows, int cols, int dtype, cudaStream_t s);
void swiglu_bwd(const void* dout, const void* gate, const void* up, void* dgate, void* dup, int64_t rows, int cols,
                int dtype, cudaStream_t s);
// rotary embedding on [tokens, heads, dim]; cos/sin are fp32 [positions, dim/2]; pos_ids may be null (pos = token % seq)
void rope_apply(const void* x, void* y, const float* cos_t, const float* sin_t, const int64_t* pos_ids, int64_t tokens,
                int seq, int heads, int dim, int neox, int backward, int dtype, int64_t row_stride, cudaStream_t s);
// y = a + b (residual add), vectorised
void add_fwd(const void* a, const void* b, void* y, int64_t n, int dtype, cudaStream_t s);

// ---- fused_dropout.cu -----------------------------------------------------------------------------------------
// out = dropout(x + bias[col]) * scale + y (bias / y optional), mask: 1 byte per element; Philox(seed, vector index, offset)
void bias_dropout_add_fwd(const void* x, const void* bias, const void* y, void* out, uint8_t* mask, int64_t n, int cols, float p, int upscale, uint64_t seed,
                          uint64_t offset, int dtype, cudaStream_t s);
void dropout_bwd(const void* dout, const uint8_t* mask, void* dx, int64_t n, float p, int upscale, int dtype, cudaStream_t s);
// act: 0 gelu, 1 relu, 2 silu; gated: out[r, c] = act(x[r, c] + b[c]) * (x[r, cols/2 + c] + b[cols/2 + c])
void bias_act_fwd(const void* x, const void* bias, void* out, int64_t rows, int cols, int act, int gated, int dtype, cudaStream_t s);

// ---- loss.cu --------------------------------------------------------------------------------------------------
// per-row softmax cross-entropy with integer labels. loss/lse fp32 [rows].
void softmax_ce_fwd(const void* logits, const int64_t* labels, float* loss, float* lse, int64_t rows, int vocab,
                    int64_t ignore_index, int dtype, cudaStream_t s);
// dlogits = (softmax - onehot) * dloss[row]; may alias logits (in-place).
void softmax_ce_bwd(const void* logits, const int64_t* labels, const float* lse, const float* dloss, void* dlogits,
                    int64_t rows, int vocab, int64_t ignore_index, int dtype, cudaStream_t s);
// vocab-parallel pieces (c_softmax_with_cross_entropy): local max / local sumexp+target logit
void vocab_parallel_ce_stats(const void* logits, const int64_t* labels, float* row_max, int64_t rows, int vocab,
                             int dtype, cudaStream_t s);
void vocab_parallel_ce_sumexp(const void* logits, const int64_t* labels, const float* row_max, float* sumexp,
                              float* target_logit, int64_t rows, int vocab, int64_t vocab_start, int dtype,
                              cudaStream_t s);
void vocab_parallel_ce_bwd(const void* logits, const int64_t* labels, const float* row_max, const float* sumexp,
                           const float* dloss, void* dlogits, int64_t rows, int vocab, int64_t vocab_start,
                           int64_t ignore_index, int dtype, cudaStream_t s);

// ---- optim.cu -------------------------------------------------------------------------------------------------
struct AdamWArgs {
  float lr, beta1, beta2, eps, weight_decay;
  float bias_c1, bias_c2;      // 1 - beta^t
  const float* grad_sq_norm;   // device: global sum of squares (nullptr = no clipping)
  float max_norm;              // clip threshold (<=0: none)
  const float* found_inf;      // device flag (nullptr = none): skip update if != 0
  const float* inv_scale;      // device: 1/loss_scale (nullptr = 1)
  // device float[3] = {lr, 1 - beta1^t, 1 - beta2^t} (nullptr = use the host values above).  With it the launch has no
  // step-dependent host argument, so a captured CUDA graph of the whole training step can be replayed while lr / t change;
  // `lr` then acts as a per-slab multiplier on dyn[0].
  const float* dyn = nullptr;
};
// p (param dtype), g (grad dtype), master fp32 (may be null), m/v in `state_dtype` (fp32 or bf16)
// master_lo (optional, bf16 parameters only): split master weights - int16 residual such that fp32 master = (bf16 bits << 16) + lo
void adamw_step(void* p, const void* g, float* master, void* m, void* v, int64_t n, int p_dtype, int g_dtype,
                int state_dtype, const AdamWArgs& a, cudaStream_t s, int16_t* master_lo = nullptr);
// accumulates sum(g^2) into *out (fp32, must be zeroed by caller) and sets *found_inf if any non-finite
void grad_sq_norm(const void* g, int64_t n, int dtype, float* out, float* found_inf, cudaStream_t s);
// g *= *scale_dev (unscale / clip by precomputed coefficient)
void scale_inplace(void* g, int64_t n, int dtype, const float* scale_dev, float scale_host, cudaStream_t s);
void sgd_momentum_step(void* p, const void* g, float* master, void* mom, int64_t n, int p_dtype, int g_dtype, float lr,
                       float momentum, float weight_decay, int nesterov, cudaStream_t s);
void lamb_stage1(const void* p, const void* g, const float* master, void* m, void* v, float* update, int64_t n,
                 int p_dtype, int g_dtype, float beta1, float beta2, float eps, float weight_decay, float bias_c1,
                 float bias_c2, float* p_sq, float* u_sq, cudaStream_t s);
void lamb_stage2(void* p, float* master, const float* update, int64_t n, int p_dtype, float lr, const float* p_sq,
                 const float* u_sq, cudaStream_t s);

// ---- moe.cu (routing on the device) ------------------------------------------------------------------------------
void moe_number_count(const int64_t* idx, int64_t n, int64_t* counts, int upper, cudaStream_t s);
void moe_assign_pos(const int64_t* idx, int64_t n, int64_t* cursor, int64_t* pos, cudaStream_t s);
void moe_limit_by_capacity(const int64_t* ec, const int64_t* cap, int64_t* out, int n_expert, int n_worker, cudaStream_t s);
void moe_prune_gate(const int64_t* idx, int64_t n, int64_t* remaining, int64_t* out, cudaStream_t s);
void moe_plan(const int64_t* counts, int n_expert, int n_tiles, int* seg_start, int* cursor, int* tile_expert, int* k0, int* kb, cudaStream_t s);
void moe_dest(const int64_t* idx, int64_t n, int* cursor, int* dest, cudaStream_t s);
void moe_rows_scatter(const void* src, const int* dest, const float* scale, int64_t n_slots, int topk, int d, void* dst, int dtype, cudaStream_t s);
void moe_rows_combine(const void* src, const int* dest, const float* w, int64_t n_tok, int topk, int d, void* out, int dtype, cudaStream_t s);
void moe_rows_dot(const void* src, const int* dest, const void* g, int64_t n_slots, int topk, int d, float* dw, int dtype, cudaStream_t s);

// ---- gemm_sm100.cu --------------------------------------------------------------------------------------------
// D[M,N] = A[M,K] * B + bias, all row-major in memory.  b_is_nk: B stored [N,K] (K contiguous) else [K,N].
// a_is_km: A stored [K,M] (M contiguous) else [M,K].  epilogue: 0 none, 1 bias, 2 bias+gelu, 3 bias+relu, 4 accumulate (D += )
struct GemmArgs {
  const void* a; const void* b; void* d; const void* bias;
  int m, n, k;
  int64_t lda, ldb, ldd;
  int a_is_km, b_is_nk;
  int epilogue;
  int dtype;       // kF16 / kBF16 inputs
  int out_dtype;   // kF16 / kBF16 / kF32
  int batch;       // >1: strided batched
  int64_t stride_a, stride_b, stride_d;
  // Fused GEMM -> reduce-scatter (push): when rs_world > 1 the epilogue does not write `d`; output row r belongs to rank
  // r / rs_rows and is stored straight into that rank's staging slot over NVLink (rs_dst[owner] = peer pointer of the slot
  // reserved for THIS rank's partials, row-major [rs_rows, n]). The owner sums its `rs_world` slots afterwards
  // (comm::p2p_reduce_slots). Requires batch == 1 and m == rs_world * rs_rows.
  int rs_world = 0;
  int rs_rows = 0;
  void* rs_dst[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  // Fused all-gather -> GEMM: `a` is the LOCAL gathered buffer [ag_world*ag_rows, k] (row-major, lda == k) of which only
  // rank ag_rank's row shard is valid at launch; one warp per CTA pulls the other shards from ag_src[r] (peer pointers to
  // each rank's shard) over NVLink while the tensor cores start on the local rows; ag_flags = zeroed uint32 counters
  // (one per 128-row block + 1); ag_pad[r] = signal pad of rank r; ag_epoch = fresh epoch of this call.
  int ag_world = 0, ag_rank = 0, ag_rows = 0;
  const void* ag_src[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  void* ag_pad[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  void* ag_flags = nullptr;
  uint32_t ag_epoch = 0;
  // Grouped GEMM over stacked expert weights (MoE).  groups = number of experts E.
  //   grouped == 1: A = [m, k] rows grouped by expert, every 256-row block belongs to ONE expert (segments padded to 256 rows);
  //                 tile_expert[m / 256] (device int32) = expert of the block or -1 (padding past the last expert);
  //                 B = stacked weights ([E, k, n] or [E, n, k] with b_is_nk, stride_b), D = [m, n].
  //   grouped == 2: per-expert weight gradient D[e] (+)= A[rows_e, m]^T B[rows_e, n] (a_is_km, !b_is_nk): k = total rows,
  //                 expert_k0[e] / expert_kb[e] (device int32) = first row and number of 64-row blocks of expert e; D = [E, m, n].
  int grouped = 0, groups = 0;
  const int* tile_expert = nullptr;
  const int* expert_k0 = nullptr;
  const int* expert_kb = nullptr;
};
// returns 0 on success, nonzero if the shape is unsupported (the binding raises)
int gemm_tcgen05(const GemmArgs& g, cudaStream_t s);
int gemm_tcgen05_supported(int m, int n, int k, int64_t lda, int64_t ldb, int64_t ldd, int a_is_km, int b_is_nk);

// ---- gemm_fp8_sm100.cu ----------------------------------------------------------------------------------------
// D[M,N] = act(scale * (A[M,K] * B[N,K]^T) + bias): A, B fp8 (E4M3 or E5M2, 1 byte, K contiguous); D bf16 / fp16 / fp32.
struct GemmFp8Args {
  const void* a; const void* b; void* d; const void* bias;   // bias in the output dtype (or nullptr)
  int m, n, k;
  int64_t lda, ldb, ldd;
  int a_e5m2, b_e5m2;
  float scale;
  const float* scale_a_dev = nullptr;   // device scalars multiplied into the dequantisation scale (quantize_fp8 outputs)
  const float* scale_b_dev = nullptr;
  const uint8_t* sfa = nullptr;         // MX block scaling: E8M0 scale blocks of A / B (mx_quantize layout); both or neither
  const uint8_t* sfb = nullptr;
  int act;          // 0 none, 1 gelu, 2 relu
  int out_dtype;
  int batch;
  int64_t stride_a, stride_b, stride_d;
};
int gemm_fp8_tcgen05(const GemmFp8Args& g, cudaStream_t s);
// OCP MX quantisation of a contiguous [rows, k] tensor along k: q = e4m3(x / 2^e), one E8M0 byte (e + 127) per 32 elements, written in
// the 512-byte block layout [rows / 128][k / 128][(row % 32) * 16 + ((row % 128) / 32) * 4 + (k / 32) % 4] the block-scaled MMA consumes.
int mx_quantize(const void* x, int64_t rows, int64_t k, int dtype, void* q, uint8_t* sf, cudaStream_t s);
int mx_dequantize(const void* q, const uint8_t* sf, int64_t rows, int64_t k, float* out, cudaStream_t s);
// ---- quant_fp8.cu: fused per-tensor fp8 quantisation ----------------------------------------------------------
// amax[0] = max(amax[0], max |x|)  (amax is a device float, zero it first)
void fp8_amax(const void* x, int64_t n, int dtype, float* amax, cudaStream_t s);
// q[M,K] (and qT[K,M] when non-null) = saturate_fp8(x * fmax / amax); inv_scale[0] = amax / fmax.  M, K multiples of 64.
void fp8_cast_transpose(const void* x, int64_t m, int64_t k, int dtype, const float* amax, int e5m2, void* q, void* qT, float* inv_scale, cudaStream_t s);

// ---- gemm_wo_sm100.cu: weight-only quantised GEMM (dequantisation inside the SM) ---------------------------------
// out[m, n] = x[m, k] @ dequant(w)[n, k]^T * scale[n] (+ bias[n]).  w: int8 [n, k] or packed int4 [n, k / 2] (low nibble = even k).
struct WoGemmArgs {
  const void* x; const void* w; const float* scale; const void* bias; void* out;
  int m, n, k;
  int int4, bf16;   // weight format; activation dtype (1 bf16, 0 fp16)
};
int gemm_weight_only(const WoGemmArgs& g, cudaStream_t s);

// ---- decode_attention.cu --------------------------------------------------------------------------------------
// Single-token decode attention: q [B,H,128], k/v cache [B,Hkv,S_max,128], lens[b] valid positions; out [B,H,128].
// part_acc: fp32 [B,H,splits,128] scratch, part_ml: fp32 [B,H,splits,2] scratch.
int decode_attention_splits(int b, int h, int smax);
int decode_attention(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* out, float* part_acc, float* part_ml, int b,
                     int h, int hkv, int smax, int d, int splits, float scale, int dtype, cudaStream_t s, const int* block_tables = nullptr,
                     int max_blocks = 0, int block_size = 0);   // block_tables: paged caches [num_blocks, Hkv, block_size, D]
// The same over paged 8-bit caches (kv_dtype kI8 / kE4M3, q fp16 / bf16): k_dq / v_dq fp32 [Hkv] dequant scales on the device.
int decode_attention_paged_q8(const void* q, const void* k_cache, const void* v_cache, const int* lens, void* out, float* part_acc, float* part_ml,
                              int b, int h, int hkv, int d, int splits, float scale, int dtype, int kv_dtype, const float* k_dq, const float* v_dq,
                              const int* block_tables, int max_blocks, int block_size, cudaStream_t s);
// Multi-token paged decode (verify rows of speculative decoding): sequence i brings n_q[i] new tokens at packed rows cu_q[i] ... over
// past[i] cached positions (the new K / V already written); key j is visible to new token r iff j <= past[i] + r.  q: [t, h, 128] rows
// (strides q_st, q_sh); out [t, h * 128] (row stride o_st), written only at the new tokens' rows; sequences with n_q = 0 are skipped.
// n_q * (h / hkv) must not exceed 64: a sequence beyond that gets NaN rows.  Caches [num_blocks, hkv, block_size, 128] of q's dtype, or
// int8 / fp8 e4m3 (kv_dtype kI8 / kE4M3) with fp32 [hkv] dequant scales.  part_acc: fp32 [b, hkv, splits, 64, 128] and part_ml: fp32
// [b, hkv, splits, 64, 2] scratch.  No host read of the lengths.
struct PagedMultiArgs {
  const void* q; const void* k_cache; const void* v_cache; void* out;
  float* part_acc; float* part_ml;
  const int* block_tables; const int* cu_q; const int* n_q; const int* past;
  int64_t q_st, q_sh, o_st;
  int b, h, hkv, d, max_blocks, block_size, splits;
  float scale;
  int dtype;
  int kv_dtype = -1;
  const float* k_dq = nullptr;
  const float* v_dq = nullptr;
};
int decode_attention_paged_multi(const PagedMultiArgs& a, cudaStream_t s);

// ---- kv_cache_quant.cu ----------------------------------------------------------------------------------------
// Quantizing write of every sequence's new K / V rows (read in place from the packed qkv [t, (h + 2 hkv) * 128] rows, row stride in
// elements) into paged 8-bit caches [num_blocks, hkv, block_size, 128].  cu_q int32 [b + 1]; enc / dec int32 [b] (a sequence with
// enc > 0 starts at position 0, otherwise at dec); quant scales fp32 [hkv].  See include/b200_kv8.cuh for the rounding rules.
struct PagedKvWriteArgs {
  const void* qkv; void* k_cache; void* v_cache;
  int64_t row_stride;
  int t, h, hkv, d, b, block_size, max_blocks;
  const int* cu_q; const int* enc; const int* dec; const int* block_tables;
  const float* k_quant_scales; const float* v_quant_scales;
  int round_type;
  float max_bound, min_bound;
  int dtype, kv_dtype;
};
int paged_kv_cache_write(const PagedKvWriteArgs& a, cudaStream_t s);

// ---- attention_sm100.cu ---------------------------------------------------------------------------------------
// Flash-attention forward (head_dim 128, fp16/bf16). q [B,Sq,H,D], k/v [B,Sk,Hk,D], o [B,Sq,H,D] as strided views (element
// strides given as {batch, seq, head}; the head_dim stride must be 1). lse: fp32 [B,H,Sq] (natural log) or nullptr.
struct AttnArgs {
  const void* q; const void* k; const void* v; void* o; float* lse;
  int b, sq, sk, h, hk, d;
  int64_t q_strides[3], k_strides[3], v_strides[3], o_strides[3];
  float scale;
  int causal;      // bottom-right aligned: key j visible to query i iff j <= i + (sk - sq)
  int dtype;
  // Column-wise row-range mask (flashmask / packed variable-length sequences): per (batch, mask head, key) an int4
  // {lt_start, lt_end, ut_start, ut_end}; query row i does NOT see key j iff lt_start <= i < lt_end or ut_start <= i < ut_end.
  // colmask == nullptr: no mask.  mask_heads is 1 (shared by all heads) or h.
  const int* colmask = nullptr;
  int mask_heads = 1;
};
int attention_fwd_supported(const AttnArgs& a);
int attention_fwd(const AttnArgs& a, cudaStream_t s);
// Causal prefill over a paged KV cache: the queries are the n_q[i] new tokens of sequence i at packed rows cu_q[i] ..., its keys are the
// past[i] + n_q[i] cached positions (the new K / V already written), read through block_tables [b, max_blocks]; key j is visible to new
// row r iff j <= past[i] + r.  q: [t, H, D] rows (strides token, head); caches [num_blocks, Hk, block_size, D] contiguous, block_size
// in {16, 32, 64, 128, 256}; o: [t, H, D] rows (strides token, head), written only at the new tokens' rows.  lse: fp32 [H, t] or
// nullptr.  Sequences with n_q = 0 are skipped.  scratch: int32 [attention_paged_prefill_scratch_ints(t, b)], 8-byte aligned.
// No host read of the lengths: the work list is built on the device.
struct PagedAttnArgs {
  const void* q; const void* k_cache; const void* v_cache; void* o; float* lse;
  int t, h, hk, d, b, num_blocks, block_size, max_blocks;
  int64_t q_strides[2], o_strides[2];
  const int* block_tables; const int* cu_q; const int* n_q; const int* past;
  int* scratch;
  float scale;
  int dtype;
  // 8-bit caches: kv_dtype kI8 / kE4M3 with fp32 [hk] dequant scales on the device (q and o stay fp16 / bf16); -1: caches of `dtype`
  int kv_dtype = -1;
  const float* k_dq = nullptr;
  const float* v_dq = nullptr;
};
int attention_paged_prefill_slots(int t, int b);
int attention_paged_prefill_scratch_ints(int t, int b);
int attention_paged_prefill_supported(const PagedAttnArgs& a);
int attention_paged_prefill(const PagedAttnArgs& a, cudaStream_t s);
// Backward (attention_bwd_sm100.cu). fwd: the forward's arguments with o (contiguous [B,Sq,H,D]) and lse filled in.
// d_o: contiguous [B,Sq,H,D]; delta: fp32 scratch [B,H,Sq]; dq: fp32 [B,Sq,H,D], every element written; dk/dv: [B,Sk,Hk,D] views (dkv_strides).
struct AttnBwdArgs {
  AttnArgs fwd;
  const void* d_o;
  float* delta;
  float* dq;
  void* dk;
  void* dv;
  int64_t dkv_strides[3];   // element strides (batch, seq, head) of dk and dv (16-byte aligned rows)
  int64_t o_strides[3];     // element strides (batch, seq, head) shared by the forward output `fwd.o` and d_o
  int64_t dq_strides[3];    // element strides (batch, seq, head) of the fp32 dq accumulator
};
int attention_bwd(const AttnBwdArgs& a, cudaStream_t s);

}  // namespace b200
