// Host-side launcher declarations for the edl_b200 sm_90a kernels.
// Kernels live in torch-free .cu files; bindings.cpp adapts torch tensors to these entry points.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace edl {

// ---- dropout masks (philox.cuh): one (seed, offset) pair per dropout site, drawn from torch's CUDA generator by the
// bindings.  Element n of the site is kept iff word n % 4 of Philox4x32-10(key = seed, counter = (n / 4, offset)) is
// >= threshold = floor(p * 2^32); a kept element is scaled by scale = fp32(1 / (1 - p)).  Under CUDA-graph capture the
// seed and offset are read at run time from seed_ptr and offset_ptr (+ offset_intragraph), so every replay draws anew.
struct PhiloxArgs {
  uint64_t seed = 0;
  uint64_t offset = 0;
  const int64_t* seed_ptr = nullptr;     // captured: the seed lives here
  const int64_t* offset_ptr = nullptr;   // captured: the offset is *offset_ptr + offset_intragraph
  uint64_t offset_intragraph = 0;
  uint32_t threshold = 0;
  float scale = 1.f;
};
// y = Z o x over n bf16 elements (dropout.cu); any n, any 2-byte alignment
void dropout_apply(const void* x, void* y, int64_t n, const PhiloxArgs& drop, cudaStream_t s);

// ---- bn.cu ----
void bn_stats(const void* x, float* sums, int64_t M, int C, cudaStream_t stream);
// mask (optional, residual + ReLU only): also write the ReLU mask bits uint8 [M, C / 8] of the stored output; needs
// bn_relu_mask_supported(M, C)
void bn_apply(const void* x, const void* res, void* y, void* mask, const float* sums, const float* gamma,
              const float* beta, float* running_mean, float* running_var, float* saved_mean,
              float* saved_rstd, int64_t M, int C, float eps, float momentum, bool relu,
              cudaStream_t stream);
void scale_shift_act(const void* x, const void* res, void* y, const float* scale,
                     const float* shift, int64_t M, int C, bool relu, cudaStream_t stream);
// ReLU mask: from the mask bits if given, else from y > 0 if given, else recomputed from x (no residual case)
void bn_bwd_reduce(const void* dy, const void* x, const void* y, const void* mask, const float* gamma,
                   const float* beta, const float* saved_mean, const float* saved_rstd,
                   float* dsums, int64_t M, int C, bool relu, cudaStream_t stream);
void bn_bwd_apply(const void* dy, const void* x, const void* y, const void* mask, const float* gamma,
                  const float* beta, const float* saved_mean, const float* saved_rstd,
                  const float* dsums, void* dx, void* dres, float* dgamma, float* dbeta, int64_t M,
                  int C, bool relu, bool accumulate, cudaStream_t stream);
// the streaming kernels run (bn_set_stream_kernels) and can write / read mask bits for this shape
bool bn_relu_mask_supported(int64_t M, int C);

// ---- bn_stream.cu (cp.async.bulk + mbarrier streaming variants; used when supported) ----
bool bn_stream_supported(int64_t M, int C);
bool bn_mask_supported(int64_t M, int C);     // bn_stream_supported and C % 128 == 0
void bn_stats_stream(const void* x, float* sums, int64_t M, int C, cudaStream_t s);
void bn_apply_stream(const void* x, const void* res, void* y, void* mask, const float* sums, const float* gamma,
                     const float* beta, float* running_mean, float* running_var, float* saved_mean,
                     float* saved_rstd, int64_t M, int C, float eps, float momentum, bool relu,
                     cudaStream_t s);
void bn_bwd_reduce_stream(const void* dy, const void* x, const void* y, const void* mask, const float* gamma,
                          const float* beta, const float* saved_mean, const float* saved_rstd,
                          float* dsums, int64_t M, int C, bool relu, cudaStream_t s);
void bn_bwd_apply_stream(const void* dy, const void* x, const void* y, const void* mask, const float* gamma,
                         const float* beta, const float* saved_mean, const float* saved_rstd,
                         const float* dsums, void* dx, void* dres, float* dgamma, float* dbeta,
                         int64_t M, int C, bool relu, bool accumulate, cudaStream_t s);
void bn_set_stream_kernels(bool enabled);

// ---- bn_fused.cu (SM-resident single-launch BN forward / backward with a grid barrier) ----
bool bn_fused_fits(int64_t M, int C, int num_operands);
const char* bn_fwd_fused(const void* x, const void* res, void* y, float* sums, const float* gamma,
                         const float* beta, float* running_mean, float* running_var,
                         float* saved_mean, float* saved_rstd, int64_t M, int C, float eps,
                         float momentum, bool relu, unsigned int* sync_counter, cudaStream_t s);
const char* bn_bwd_fused(const void* dy, const void* x, const void* y, const float* gamma,
                         const float* beta, const float* saved_mean, const float* saved_rstd,
                         float* dsums, void* dx, void* dres, float* dgamma, float* dbeta, int64_t M,
                         int C, bool relu, bool accumulate, unsigned int* sync_counter,
                         cudaStream_t s);  // runtime switch (A/B measurements); default on

// ---- runtime policy (bn.cu): keep every SM in the max-shared-memory carveout so that kernels with
// large dynamic smem (TMA rings, GEMM stages) never force an L1/smem re-partition between launches ----
void set_smem_carveout_policy(bool prefer_max_shared);
bool smem_carveout_policy();
void apply_carveout(const void* kernel);   // call after cudaFuncSetAttribute(MaxDynamicSharedMemorySize)

// ---- optim.cu ----
void sgd_momentum(void* param_lp, float* master, float* mom, const void* grad, bool grad_is_bf16,
                  const float* wd_mask, int64_t n, const float* lr, const float* grad_scale,
                  const int* found_inf, float momentum, float wd, bool nesterov,
                  cudaStream_t stream);
void adam_step(void* param_lp, float* master, float* m, float* v, const void* grad,
               bool grad_is_bf16, int64_t n, const float* lr, const float* grad_scale,
               const int* found_inf, const float* step, float beta1, float beta2, float eps,
               float wd, bool decoupled, cudaStream_t stream);

// sum(g^2) of a flat gradient buffer into *out (+=), and the global-norm clip factor
//   grad_scale = min(1, max_norm / (sqrt(sum of parts) + 1e-6))   (parts: one squared-norm partial per rank)
void grad_sqnorm(const void* grad, bool grad_is_bf16, int64_t n, float* out, cudaStream_t stream);
void clip_scale(const float* parts, int nparts, int stride, float max_norm, float* grad_scale, float* norm_out,
                cudaStream_t stream);

// ---- loss.cu ----
void soft_ce_fwd(const void* logits, bool logits_bf16, const void* target, bool target_bf16,
                 const int64_t* labels, float* loss_out, float* row_stats, int N, int C, int mode,
                 float s_temp, float t_temp, float label_smooth, bool kl, float loss_scale,
                 cudaStream_t stream);
void soft_ce_bwd(const void* logits, bool logits_bf16, const void* target, bool target_bf16,
                 const int64_t* labels, const float* row_stats, const float* grad_out,
                 void* dlogits, int N, int C, int mode, float s_temp, float t_temp,
                 float label_smooth, float loss_scale, cudaStream_t stream);
void topk_acc(const void* logits, bool logits_bf16, const int64_t* labels, float* counts, int N,
              int C, cudaStream_t stream);

// ---- pool.cu ----
void maxpool3x3s2_fwd(const void* x, void* y, uint8_t* idx, int N, int H, int W, int C,
                      cudaStream_t s);
void maxpool3x3s2_bwd(const void* dy, const uint8_t* idx, void* dx, int N, int H, int W, int C,
                      cudaStream_t s);
void avgpool2x2_fwd(const void* x, void* y, int N, int H, int W, int C, cudaStream_t s);
void avgpool2x2_bwd(const void* dy, void* dx, int N, int H, int W, int C, cudaStream_t s);
void dilate2(const void* x, void* y, int N, int H, int W, int C, cudaStream_t s);   // zero-insertion by 2 (NHWC bf16)
void gap_fwd(const void* x, void* y, int N, int HW, int C, cudaStream_t s);
void gap_bwd(const void* dy, void* dx, int N, int HW, int C, cudaStream_t s);

// ---- allreduce.cu ----
struct CommHandles {
  void* data[16];
  void* sig[16];
  void* mc_data;
  int rank;
  int world;
  unsigned long long timeout_ns;
};
int comm_sig_words();
int comm_max_world();
int comm_error_word_offset();
void allreduce_oneshot(const CommHandles& h, void* out, bool is_bf16, int64_t n, float scale,
                       int* found_inf, float* sqnorm, int nblocks, cudaStream_t stream);
void allreduce_twoshot(const CommHandles& h, bool is_bf16, int64_t n, float scale, int* found_inf,
                       float* sqnorm, bool multimem, int nblocks, cudaStream_t stream);
// fused reduce-scatter -> SGD-momentum -> parameter all-gather of one bf16 bucket (allreduce.cu)
void allreduce_sgd(const CommHandles& h, void* const* param_ptrs, void* mc_param, float* master, float* mom,
                   const float* wd_mask, int64_t n, float scale, int* found_inf_out, float* sqnorm,
                   const float* lr, const int* skip_flag, float momentum, float wd, bool nesterov, bool multimem,
                   int nblocks, cudaStream_t stream);
void comm_broadcast(const CommHandles& h, int root, int64_t nbytes, int nblocks,
                    cudaStream_t stream);
void comm_allgather_scalars(const CommHandles& h, const float* in, float* out, int count,
                            cudaStream_t stream);

// ---- misc.cu ----
void rope(const void* x, const float* cosv, const float* sinv, void* y, int64_t T, int H, int D,
          bool inverse, cudaStream_t s);
// pixel-pair form of the 32-channel 3x3 stem convolutions (misc.cu): W [cout,3,3,32] <-> W2 [2*cout,3,3,64]
void pair_weight_expand(const void* w, void* w2, int cout, cudaStream_t s);
void pair_weight_fold(const void* dw2, void* dw, int cout, bool accumulate, cudaStream_t s);
void fold_pair_stats(const float* s2, float* stats, int cout, cudaStream_t s);
// ---- stem.cu: first stem convolution (3 -> 32, 3x3 / stride 2 / pad 1, NHWC bf16) + BN statistics of its output ----
void stem_conv3x3s2(const void* x, const void* w, void* y, float* stats, int N, int H, int W, cudaStream_t s);
// its weight gradient: dw KRSC [32,3,3,3] bf16 (+)= ; ws: >= 864 zero floats (left zero), counter: one zero int (left zero)
// A [N * Ho * Wo, 160] bf16 = im2col of the 7x7 / stride 2 / pad 3 convolution of x [N, H, W, 3] ((r, s, c) order, zero-padded)
const char* stem7_im2col(const void* x, void* a, int N, int H, int W, cudaStream_t s);
const char* stem_wgrad(const void* x, const void* dy, float* ws, int* counter, void* dw, bool accumulate, int N, int H,
                       int W, cudaStream_t s);

void embedding_bag_fwd(const void* table, bool bf16, const int64_t* ids, void* out, int64_t B, int L,
                       int D, cudaStream_t s);
void embedding_bag_bwd(const void* dout, bool bf16, const int64_t* ids, float* dtable, int64_t B, int L,
                       int D, cudaStream_t s);
void normalize_u8(const uint8_t* x, void* y, int64_t N, int H, int W, const float* mean,
                  const float* stdv, const uint8_t* flip, cudaStream_t s);

// ---- embedding.cu: row-sparse embedding bags (fp32 tables) ----
// offsets == nullptr: fixed-length bags [B, L]; else CSR bag starts [B] over ids [nnz] (nn.EmbeddingBag convention)
void embedding_bag_mean_fwd(const float* table, const int64_t* ids, const int64_t* offsets, float* out, int64_t B,
                            int64_t nnz, int L, int D, cudaStream_t s);
// uncoalesced row-sparse gradient: indices [nnz], values [nnz, D]
void embedding_bag_mean_bwd_sparse(const float* dout, const int64_t* ids, const int64_t* offsets, int64_t* indices,
                                   float* values, int64_t B, int64_t nnz, int L, int D, cudaStream_t s);
// the same for S slots of fixed-length bags at once: ids [B, S, L], slot s reads table w[s] (all of width D);
// out [B, S, D]; backward: indices [S, B * L], values [S, B * L, D] (slot-major)
constexpr int kMaxSparseTables = 64;
struct SlotTables {
  const float* w[kMaxSparseTables];
};
void embedding_bags_mean_fwd(const int64_t* ids, float* out, int64_t B, int S, int L, int D, const SlotTables& tabs,
                             cudaStream_t s);
void embedding_bags_mean_bwd_sparse(const float* dout, const int64_t* ids, int64_t* indices, float* values, int64_t B,
                                    int S, int L, int D, cudaStream_t s);
// lazy Adam over the rows of the row-sparse gradients of up to kMaxSparseTables fp32 tables [rows, D] of one width D
struct SparseTables {
  float* w[kMaxSparseTables];
  float* m[kMaxSparseTables];
  float* v[kMaxSparseTables];
  int64_t rows[kMaxSparseTables];
  int64_t start[kMaxSparseTables];   // first position of table t's rows in the concatenated gradient
  int count;
};
// keys[i] = t << 40 | ids[i] for the concatenated gradient indices (-1: id outside its table)
void sparse_adam_keys(const int64_t* ids, int64_t* keys, int64_t n, const SparseTables& tabs, cudaStream_t s);
// sorted_keys / perm: stable sort of the keys; values: the concatenated gradient rows [n, D]
void sparse_adam(const int64_t* sorted_keys, const int64_t* perm, const float* values, int64_t n, int D,
                 const SparseTables& tabs, const float* lr, const float* step, float beta1, float beta2, float eps,
                 cudaStream_t s);

// ---- augment.cu: random-resized crop + flip + normalise from decoded uint8 RGB images of different sizes ----
struct AugmentItem {   // one per output image; 32 bytes = 8 x int32 (the Python side fills an int32 [N, 8] tensor)
  int64_t offset;      // byte offset of the decoded image (interleaved RGB) inside the pool buffer
  int pitch;           // bytes per source row
  int y, x, ch, cw;    // crop box inside the source image
  int flip;            // mirror horizontally
};
void crop_resize_normalize(const uint8_t* pool, const AugmentItem* items, void* y, int N, int S, const float* mean,
                           const float* stdv, cudaStream_t s);

// ---- logit_ship.cu (teacher -> student over NVSwitch peer memory, fused with the loss) ----
void peer_ship(const void* src, void* dst_peer, int64_t nbytes, void* flag_peer, const void* seq_ptr,
               uint32_t seq_imm, void* done_counter, cudaStream_t s);
void logit_ship(const void* logits, void* slot_peer, float* stats_peer, int B, int C, float temperature,
                void* flag_peer, const void* seq_ptr, uint32_t seq_imm, void* done_counter,
                cudaStream_t s);
void soft_ce_recv(const void* logits, bool logits_bf16, const void* slot, const float* slot_stats,
                  const void* flag, const void* seq_ptr, uint32_t seq_imm, float* loss_out,
                  float* row_stats, int B, int C, float s_temp, float t_temp, bool kl, float loss_scale,
                  double timeout_s, void* err, cudaStream_t s);
void slot_ack(void* ack_peer, const void* seq_ptr, uint32_t seq_imm, cudaStream_t s);
void wait_flag_async(const void* flag, const void* seq_ptr, uint32_t seq_imm, double timeout_s, void* err,
                     cudaStream_t s);

// ---- attention.cu / layernorm.cu: the Transformer encoder of the NLP teacher (inference) ----
constexpr int kAttnMaxLen = 512;
bool attention_supported(int B, int L, int H, int head_dim);
// qkv bf16 [B * L, 3 * H * 64] (Q | K | V column blocks, 16-byte aligned), mask uint8 [B, L] (1 = attend; nullptr: all),
// out bf16 [B * L, H * 64].  lse: nullptr, or fp32 [B, H, L] that receives what the backward needs to recompute the
// probabilities (attention.cu).  drop (training, with lse): dropout on the probabilities, element (b, h, i, j) at flat
// index ((b H + h) L + i) L + j of the mask.  Returns nullptr or an error string.
const char* attention_fwd(const void* qkv, const uint8_t* mask, void* out, int B, int L, int H, cudaStream_t stream,
                          float* lse = nullptr, const PhiloxArgs* drop = nullptr);
// Backward of attention_fwd (attention_bwd.cu): from qkv, the forward's out and lse and the output gradient dout
// (bf16 [B * L, H * 64]) writes dqkv bf16 [B * L, 3 * H * 64] (dQ | dK | dV in the layout of qkv).  delta: fp32 [B, H, L]
// workspace.  drop: the forward's dropout (the same mask is regenerated).  Deterministic, no atomics.
const char* attention_bwd(const void* qkv, const uint8_t* mask, const void* out, const float* lse, const void* dout,
                          void* dqkv, float* delta, int B, int L, int H, cudaStream_t stream,
                          const PhiloxArgs* drop = nullptr);
bool attention_varlen_supported(int T, int B, int max_len, int H, int head_dim);
// Packed sequences: qkv bf16 [T, 3 * H * 64], sequence b in rows [cu_seqlens[b], cu_seqlens[b + 1]) (int32 device
// offsets, 1 <= length <= max_len <= 512), key_mask uint8 [T] (1 = attend; nullptr: all), out bf16 [T, H * 64];
// maps: device workspace of 2 * B CUtensorMaps (64-byte aligned).  A sequence's output depends on its own rows only.
// lse (training): nullptr, or fp32 [H, T] that receives lse at h * T + packed row (a separate kernel instantiation; the
// inference one is unchanged).  drop (training, with lse): dropout on the probabilities, element (b, h, i, j) at flat
// index ((b H + h) 512 + i) 512 + j of the mask: the fixed stride kAttnMaxLen keeps the sequences' ranges disjoint.
const char* attention_varlen_fwd(const void* qkv, const int* cu_seqlens, const uint8_t* key_mask, void* out, void* maps,
                                 int T, int B, int max_len, int H, cudaStream_t stream, float* lse = nullptr,
                                 const PhiloxArgs* drop = nullptr);
// Backward of the packed training forward (attention_bwd.cu): from qkv, out and lse [H, T] of attention_varlen_fwd and
// dout bf16 [T, H * 64], writes the rows of every sequence of dqkv bf16 [T, 3 * H * 64] (rows outside all sequences are
// not written).  delta: fp32 [H, T] workspace.  drop: the forward's dropout.  A sequence's gradients depend on its own
// rows only.  Deterministic, no atomics, no host synchronisation.
const char* attention_varlen_bwd(const void* qkv, const int* cu_seqlens, const uint8_t* key_mask, const void* out,
                                 const float* lse, const void* dout, void* dqkv, float* delta, int T, int B, int max_len,
                                 int H, cudaStream_t stream, const PhiloxArgs* drop = nullptr);
constexpr int kLnMaxC = 1024;
bool layernorm_supported(int C);
// y[r] = (x[r] - mean) * rsqrt(var + eps) * gamma + beta over the C columns of each row; x, y bf16 [rows, C] (row pitch
// C), gamma / beta fp32 [C]; statistics in fp32
void layernorm_fwd(const void* x, const float* gamma, const float* beta, void* y, int64_t rows, int C, float eps,
                   cudaStream_t s);
// the same over x[r] = word[ids[r]] + pos[pos_ids[r]] + seg[seg_ids[r]] (bf16 tables [*, C], sum in fp32).  An id
// outside its table reads nothing (the row sums the other tables) and sets *err to 1.  drop (training): dropout on the
// output, element (r, c) at flat index r * C + c of the mask.
void embedding_layernorm_fwd(const int64_t* ids, const int64_t* pos_ids, const int64_t* seg_ids, const void* word,
                             int64_t n_word, const void* pos, int64_t n_pos, const void* seg, int64_t n_seg,
                             const float* gamma, const float* beta, void* y, int64_t rows, int C, float eps, int* err,
                             cudaStream_t s, const PhiloxArgs* drop = nullptr);
// Quantising variants: also q e4m3 [rows, C] (contiguous, 8-byte aligned) and sa fp32 [ceil(C/128), rows] of the stored
// bf16 y, bit for bit what quantize_e4m3_blocks (gemm.h) makes of y: s = max|y| / 448 per row and 128-column block (1
// for an all-zero block), q = sat(y / s).
void layernorm_e4m3_fwd(const void* x, const float* gamma, const float* beta, void* y, void* q, float* sa, int64_t rows,
                        int C, float eps, cudaStream_t s);
void embedding_layernorm_e4m3_fwd(const int64_t* ids, const int64_t* pos_ids, const int64_t* seg_ids, const void* word,
                                  int64_t n_word, const void* pos, int64_t n_pos, const void* seg, int64_t n_seg,
                                  const float* gamma, const float* beta, void* y, void* q, float* sa, int64_t rows, int C,
                                  float eps, int* err, cudaStream_t s);
// Backward of layernorm_fwd from the saved pre-LN input x (statistics recomputed): dx bf16 [rows, C]; per-CTA fp32
// partials of dgamma / dbeta in part [layernorm_bwd_ctas(rows), 2, C], reduced in a fixed order into dgamma, dbeta [C].
int layernorm_bwd_ctas(int64_t rows);
void layernorm_bwd(const void* x, const void* dy, const float* gamma, void* dx, float* part, float* dgamma,
                   float* dbeta, int64_t rows, int C, float eps, cudaStream_t s);
// Backward of embedding_layernorm_fwd: re-gathers the row sum and writes its gradient dE fp32 [rows, C] (the gradient of
// each of the three gathered table rows), plus dgamma / dbeta as in layernorm_bwd.  drop: the forward's output dropout
// (applied to dy as it is loaded).
void embedding_layernorm_bwd(const int64_t* ids, const int64_t* pos_ids, const int64_t* seg_ids, const void* word,
                             int64_t n_word, const void* pos, int64_t n_pos, const void* seg, int64_t n_seg,
                             const void* dy, const float* gamma, float* dE, float* part, float* dgamma, float* dbeta,
                             int64_t rows, int C, float eps, cudaStream_t s, const PhiloxArgs* drop = nullptr);

// ---- lstm.cu: bidirectional LSTM recurrence of the BiLSTM student (H = 128; layouts in lstm.cu's header) ----
constexpr int kLstmHidden = 128;
bool lstm_supported(int B, int L, int E, int H);
// xproj bf16 [L * B, 8H] (thread order), whh bf16 [2, 4H, H] (nn.LSTM layout, 16-byte aligned), lengths int32 [B];
// writes hs bf16 [(L + 2) * B, 2H], hn bf16 [2, B, H], gates bf16 [L * B, 2, H, 4], cs fp32 [L * B, 2, H]
const char* lstm_fwd(const void* xproj, const void* whh, const int* lengths, void* hs, void* hn, void* gates, float* cs,
                     int B, int L, cudaStream_t stream);
// dy bf16 (b, t, c) at b * dy_sb + t * dy_st + c, or nullptr (zero); dhn bf16 [2, B, H] or nullptr;
// writes dgates bf16 [L * B, 8H] (nn.LSTM row order per direction)
const char* lstm_bwd(const void* whh, const int* lengths, const void* gates, const float* cs, const void* dy,
                     int64_t dy_sb, int64_t dy_st, const void* dhn, void* dgates, int B, int L, cudaStream_t stream);

}  // namespace edl
