// Host API of the wgmma GEMM / implicit-GEMM conv kernels (gemm.cu, conv3x3.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace edl {

struct PhiloxArgs;   // kernels.h

// Fused BatchNorm-backward reduction (persistent dgrad kernels): the GEMM / conv output D is the gradient
// dy of a BN layer's output; the epilogue accumulates dsums[0:C] += sum(dy_m), dsums[C:2C] += sum(dy_m * xhat)
// (dy_m = dy masked by the layer's ReLU) so that the BN backward needs no reduction pass of its own.
struct BnBwdFuse {
  const void* x = nullptr;       // bf16, BN input (conv output), same shape / layout as D
  const void* y = nullptr;       // bf16, BN output: only for ReLU after a residual add (mask = y > 0)
  const void* mask = nullptr;    // or uint8 [M, C / 8], bit b of byte j = (y[:, 8 j + b] > 0): D is then stored masked
                                 // (1x1 dgrad, C % 128 == 0)
  const float* mean = nullptr;
  const float* rstd = nullptr;
  const float* gamma = nullptr;
  const float* beta = nullptr;
  float* dsums = nullptr;        // fp32 [2C], pre-zeroed
  bool relu = false;
};

struct GemmArgs {
  const void* A = nullptr;  // bf16
  const void* B = nullptr;  // bf16
  void* D = nullptr;        // bf16 [M, N]
  int M = 0, N = 0, K = 0;
  int64_t lda = 0, ldb = 0, ldd = 0;  // row pitches in elements of the *stored* 2-D arrays
  bool a_mn_major = false;            // A stored as [K, M] (M contiguous)
  bool b_mn_major = false;            // B stored as [K, N] (N contiguous); default B is [N, K]
  const float* col_scale = nullptr;   // per-output-column scale (folded BN) or nullptr
  const float* col_shift = nullptr;   // per-output-column shift / bias or nullptr
  bool relu = false;
  float* col_stats = nullptr;         // [2N] fp32: += sum, sum of squares of the stored outputs
  // Weight-gradient form (A and B both MN-major, N % 4 == 0): D (+= when accumulate) is written with plain 8-byte
  // stores.  With split_k > 1 the K reduction is split over CTAs: every CTA stores its fp32 partial tile into
  // partials[split][tile][128 x BLOCK_N] with plain coalesced stores and splitk_reduce sums the splits into D.  The
  // partials are required then (partials_elems >= split * tiles * 128 * BLOCK_N).
  int split_k = 1;
  bool accumulate = false;
  float* partials = nullptr;
  int64_t partials_elems = 0;
  // weight-gradient form: columns of D that are stored (0: all N).  With n_out < N the last N - n_out columns of the
  // product (zero padding of the B operand, e.g. the 7x7 stem's 147 -> 160 im2col width) never reach memory; D then
  // needs no alignment beyond its element size
  int n_out = 0;
  int device = -1;                    // CUDA device ordinal of the operands (binds the context)
  // D = A*B + add_src (bf16 [M, N], row pitch ld_add): fuses the gradient accumulation of a tensor with two
  // consumers (residual branch + 1x1 conv) into the dgrad epilogue.  Persistent kernel only.
  const void* add_src = nullptr;
  int64_t ld_add = 0;
  BnBwdFuse bn;                        // bn.x != nullptr enables the fused BN-backward reduction (row pitch = ldd)
  // D = gelu(A*B^T * col_scale + col_shift), erf form, fp32 (inference; B K-major, no addend / ReLU / statistics).
  // Persistent kernel only.
  bool gelu = false;
  // with gelu: also store the pre-activation u = A*B^T * col_scale + col_shift as bf16 [M, N] (row pitch ld_u), the
  // training forward of FFN1
  void* gelu_u = nullptr;
  int64_t ld_u = 0;
  // D = (A*B) * gelu'(add_src) in fp32 (B MN-major, add_src = u): the dgrad of FFN2 that yields dU of FFN1
  bool gelu_grad = false;
  // D = add_src + Z o (A*B^T + col_shift), Z the dropout mask of *dropout at flat index row * N + col (B K-major, an
  // addend, no scale / ReLU / statistics): the residual branch of a Transformer layer in training.  Persistent kernel only.
  const PhiloxArgs* dropout = nullptr;
  // fused "GEMM -> peer ship" (EPI 0 only): D may be a PEER GPU's buffer (NVLink-mapped address);
  // every CTA TMA-stores its tile there, and the CTA that completes last publishes
  // *ship_flag (peer address) = seq with release/system semantics -- no separate copy kernel.
  void* ship_flag = nullptr;
  const void* ship_seq_ptr = nullptr;  // device uint32 (graph-replayable) or nullptr -> ship_seq_imm
  uint32_t ship_seq_imm = 0;
  void* ship_done = nullptr;           // local zero-initialised uint32 counter (re-armed by the kernel)
};

// Returns nullptr on success, else a static error string.
const char* gemm_bf16(const GemmArgs& args, cudaStream_t stream);

// out[m0 + r][col(c)] (+)= sum over splits of partials[z][tile][r][c]; tiles are [rows x cols] fp32, tile t covers output
// rows (t / tiles_n) * rows.. and -- taps == 1 -- columns (t % tiles_n) * cols..; taps == 3 (3x3 wgrad): t = tile * 3 + r,
// column c of the tile is tap s = c / (cols / 3) of filter row r: output column (r * 3 + s) * cin + n0 + c % (cols / 3).
void splitk_reduce(const float* partials, int split, int ctas, int tiles_n, int rows, int cols, int taps, int cin,
                   int M, int N, void* out_bf16, int64_t ldo, bool accumulate, cudaStream_t stream);

// 3x3 / stride 1 / pad 1 NHWC convolution as an implicit GEMM (conv3x3.cu): nine shifted TMA tile loads
// per input-channel block (out-of-bounds rows/columns are zero-filled by the TMA unit = the padding)
// accumulate into one register tile.  `dgrad` computes the data gradient with the same kernel (mirrored
// taps, weight tile read MN-major).
struct Conv3x3Args {
  const void* X = nullptr;   // bf16 NHWC [N, H, W, Cx]  (fwd: input; dgrad: dY)
  const void* Wt = nullptr;  // bf16 KRSC [Cout, 3, 3, Cin]
  void* Y = nullptr;         // bf16 NHWC [N, H, W, Cy]  (fwd: output; dgrad: dX)
  int N = 0, H = 0, W = 0, Cin = 0, Cout = 0;
  bool dgrad = false;
  float* col_stats = nullptr;  // fwd only: [2*Cout] += per-channel sum / sum of squares of Y
  BnBwdFuse bn;                // dgrad only: fused BN-backward reduction over Y (= dX)
  // inference epilogue (fprop, persistent kernel): Y = relu?(conv * col_scale[c] + col_shift[c]) (folded BN)
  const float* col_scale = nullptr;
  const float* col_shift = nullptr;
  bool relu = false;
  int groups = 1;              // grouped fprop: Cin/groups % 64 == 0, Cout/groups == 64 or % 128 == 0; Wt is
                               // [Cout, 3, 3, Cin/groups]
  int stride = 1;              // 1 or 2 (fprop on the persistent kernel only).  N, H, W are the OUTPUT geometry; with
                               // stride 2 the input X is [N, 2H, 2W, Cin] and is sampled by the TMA traversal stride
  int ksize = 3;               // 3, or 1: the 1x1 / pad 0 / stride 2 convolution (conv1x1_s2_bf16), Wt is [Cout, Cin]
  int device = -1;
};
bool conv3x3_supported(int N, int H, int W, int Cin, int Cout, bool dgrad, int groups = 1);
const char* conv3x3_bf16(const Conv3x3Args& args, cudaStream_t stream);
// input gradient of the stride-2 convolution: args.X = dY [N, H, W, Cout], args.Y = dX [N, 2H, 2W, Cin], N/H/W of dY
bool conv3x3_dgrad_s2_supported(int N, int Ho, int Wo, int Cin, int Cout);
const char* conv3x3_dgrad_s2_bf16(const Conv3x3Args& args, cudaStream_t stream);
// 1x1 / pad 0 / stride 2 convolution = the centre tap of the 3x3 / pad 1 / stride 2 one: y[n, h, w] = x[n, 2h, 2w] * W^T.
// fprop (args.dgrad == false): X = x [N, 2H, 2W, Cin], Y = y [N, H, W, Cout] (+ col_stats or the inference epilogue);
// dgrad: X = dY [N, H, W, Cout], Y = dX [N, 2H, 2W, Cin], zero at the three pixel parities the convolution skips.
// Wt is [Cout, Cin]; N, H, W are the output geometry.  Persistent kernel only.
bool conv1x1_s2_supported(int N, int Ho, int Wo, int Cin, int Cout, bool dgrad);
const char* conv1x1_s2_bf16(const Conv3x3Args& args, cudaStream_t stream);

// Weight gradient of the same convolution (conv3x3_wgrad.cu): dW[Cout,3,3,Cin] (+)= sum_pixels dY x shifted X, pixel
// reduction split over `split_k` CTAs through partial tiles like the 1x1 weight-gradient GEMM.
struct Conv3x3WgradArgs {
  const void* X = nullptr;    // bf16 NHWC [N, H, W, Cin]   (the convolution's input)
  const void* dY = nullptr;   // bf16 NHWC [N, H, W, Cout]
  void* dW = nullptr;         // bf16 KRSC [Cout, 3, 3, Cin] (e.g. a window of the flat gradient bucket)
  int N = 0, H = 0, W = 0, Cin = 0, Cout = 0;   // H, W: OUTPUT (= dY) size; the input is stride times as large
  int split_k = 1;
  bool accumulate = false;    // dW += result instead of dW = result
  int device = -1;
  int stride = 1;             // 2: X is [N, 2H, 2W, Cin], read through the TMA traversal stride (version-1 kernel)
  int ksize = 3;              // 1: the 1x1 / pad 0 / stride 2 convolution, dW is [Cout, Cin] (version-1 kernel, one tap)
  // fp32 partial tiles [split][ctas][128 x 3*BLOCK_N], required when split_k > 1: split_k *
  // conv3x3_wgrad_tiles(Cin, Cout) * 128 * 192 elements cover both kernel versions
  float* partials = nullptr;
  int64_t partials_elems = 0;
};
bool conv3x3_wgrad_supported(int N, int H, int W, int Cin, int Cout);
bool conv3x3_wgrad_s2_supported(int N, int Ho, int Wo, int Cin, int Cout);
int conv3x3_wgrad_s2_kblocks(int N, int Ho, int Wo);
int conv3x3_wgrad_tiles(int Cin, int Cout);
int conv3x3_wgrad_ctas(int Cin, int Cout);        // (tile, filter row) CTAs per K split of the active kernel version
void set_wgrad3_version(int version, int base_offset_mode);   // 1 = three X loads per block, 2 = one haloed X load (default)
int get_wgrad3_version();
int conv3x3_wgrad_kblocks(int N, int H, int W);   // pixel blocks of the reduction (upper bound for split_k)
void conv3x3_wgrad_plan(int N, int H, int W, int* bh, int* nb, int* kb);   // pixel box {W, bh rows, nb images}, kb = W*bh*nb
const char* conv3x3_wgrad_bf16(const Conv3x3WgradArgs& args, cudaStream_t stream);

// Persistent variants (gemm_persist.cu): one CTA per SM streams tiles; the loads of the next tile overlap the epilogue.  Used by gemm_bf16 / conv3x3_bf16 when enabled (default).
int get_bnr_mode();            // fused BN-backward reduction: 2 = column loop over the staged tiles
void set_persistent_gemm(bool on);
bool persistent_gemm_enabled();
void set_persist_trace(long long* buf);   // debug: int64 [3 * 16 * 8] device buffer for clock64() phase stamps of CTA 0, or nullptr
void set_epilogue_warps(int n);      // 8 or 16 epilogue warps for the 128 / 256 column persistent kernels (EDL_EPI_WARPS)
bool conv3x3_halo_plan(int N, int H, int W, int* BH, int* BN, int* tiles_h, int* tiles_img);   // host only
void set_conv_halo(bool on);         // haloed A tiles for the 3x3 / stride 1 fprop and dgrad (default on; EDL_CONV_HALO=0)
bool get_conv_halo();
void set_conv_resident_weights(bool on);   // 64-channel layers / groups: weights resident across a CTA's run of tiles (EDL_CONV_BRES=0)
void set_wide_gemm_tiles(bool on);   // 128 x 256 tiles for large-N inference GEMMs (default on; EDL_GEMM_WIDE=0)
const char* gemm_bf16_persistent(const GemmArgs& args, cudaStream_t stream);
const char* conv3x3_dgrad_s2_persistent(const Conv3x3Args& args, int BH, int BN, int tiles_h, int tiles_img,
                                        cudaStream_t stream);
const char* conv3x3_bf16_persistent(const Conv3x3Args& args, int BH, int BN, int tiles_h, int tiles_img,
                                    cudaStream_t stream);
const char* conv1x1_dgrad_s2_persistent(const Conv3x3Args& args, int BH, int BN, int tiles_h, int tiles_img,
                                        cudaStream_t stream);

// internal: N-d bf16 tensor-map encoder shared by the TMA kernels (defined in gemm.cu)
const char* encode_tmap_bf16(void* out, const void* ptr, int rank, const uint64_t* dims,
                             const uint64_t* strides_bytes, const uint32_t* box);
const char* encode_tmap(void* out, const void* ptr, int rank, const uint64_t* dims,
                        const uint64_t* strides_bytes, const uint32_t* box, int elem_bytes);
const char* encode_tmap_strided(void* out, const void* ptr, int rank, const uint64_t* dims,
                                const uint64_t* strides_bytes, const uint32_t* box, const uint32_t* elem_strides,
                                int elem_bytes, int swizzle_bytes = 128);   // 128, 64 or 0 (none)

// FP8 (e4m3) inference GEMM (gemm_fp8.cu): D[M,N] bf16 = relu?((A[M,K] * B[N,K]^T) * col_scale[n] + col_shift[n])
// A, B e4m3 bytes, K-major; col_scale carries act_scale * weight_scale[n] (* folded BN scale).
struct GemmFp8Args {
  const void* A = nullptr;
  const void* B = nullptr;
  void* D = nullptr;
  int M = 0, N = 0, K = 0;
  int64_t lda = 0, ldb = 0, ldd = 0;   // row pitches in elements
  const float* col_scale = nullptr;
  const float* col_shift = nullptr;
  bool relu = false;
  int device = -1;
  // gemm_fp8_blockscaled only: a_scales fp32 [ceil(K/128), M], b_scales fp32 [ceil(N/128), ceil(K/128)]
  const float* a_scales = nullptr;
  const float* b_scales = nullptr;
  // gemm_fp8_blockscaled: optional bf16 addend [M, N] (row pitch ld_add elements), added after col_shift
  const void* add = nullptr;
  int64_t ld_add = 0;
  // gemm_fp8_blockscaled_gelu_e4m3 only: the output's block scales, fp32 [ceil(N/128), M]
  float* a_scales_out = nullptr;
};
const char* gemm_fp8(const GemmFp8Args& args, cudaStream_t stream);
// D[M,N] bf16 = relu?((sum_b (A_b * B_b^T) * a_scales[b, m] * b_scales[n / 128, b]) * col_scale[n] + col_shift[n]
// (+ add[m, n] when add is set)) over the 128-element K blocks b; col_scale carries only the folded BN scale here.
const char* gemm_fp8_blockscaled(const GemmFp8Args& args, cudaStream_t stream);
// FFN1 of the sequence teacher: g = bf16(gelu(sum_b (A_b * B_b^T) * a_scales[b, m] * b_scales[n / 128, b] + col_shift[n]))
// (erf form), quantised per row and 128-column block as quantize_e4m3_blocks does: D holds e4m3 bytes [M, N] (row
// pitch ldd bytes, N % 16 == 0) and a_scales_out[n / 128, m] their scales.  No col_scale, ReLU or addend.
const char* gemm_fp8_blockscaled_gelu_e4m3(const GemmFp8Args& args, cudaStream_t stream);

// bf16 -> e4m3 with a per-tensor scale (q = sat(x / scale)); amax_out (optional) receives max|x| for
// calibration / delayed scaling.
void quantize_e4m3(const void* x_bf16, void* q, int64_t n, const float* scale, float* amax_out, cudaStream_t s);

// bf16 [M, K] (row pitch lda elements) -> e4m3 q [M, K] (contiguous) and fp32 sa [ceil(K/128), M]: per row and
// 128-element K block, s = max|x| / 448 (1 when the block is all zero) and q = sat(x / s).  K % 8 == 0.
const char* quantize_e4m3_blocks(const void* x_bf16, int64_t lda, void* q, float* sa, int M, int K, cudaStream_t s);

}  // namespace edl
