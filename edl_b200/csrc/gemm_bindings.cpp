// torch bindings for the wgmma GEMM (gemm.cu).
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "gemm.h"
#include "kernels.h"

namespace {
using torch::Tensor;

template <typename T>
inline T* optp(const c10::optional<Tensor>& t) {
  return t.has_value() && t->defined() ? reinterpret_cast<T*>(t->data_ptr()) : nullptr;
}

// bn = [x, y | mask | None, mean, rstd, gamma, beta, dsums] (+ relu flag): see gemm.h BnBwdFuse.  The second entry is
// the bf16 BN output or its uint8 ReLU mask bits [M, C / 8].
edl::BnBwdFuse parse_bn(const c10::optional<std::vector<c10::optional<Tensor>>>& bn, bool relu, int64_t numel,
                        int64_t channels) {
  edl::BnBwdFuse f;
  if (!bn.has_value()) return f;
  const auto& v = *bn;
  TORCH_CHECK(v.size() == 7, "bn fuse list needs 7 entries");
  TORCH_CHECK(v[0].has_value() && v[0]->scalar_type() == at::kBFloat16 && v[0]->numel() == numel);
  f.x = v[0]->data_ptr();
  if (v[1].has_value() && v[1]->defined()) {
    if (v[1]->scalar_type() == at::kByte) {
      TORCH_CHECK(v[1]->is_contiguous() && channels % 128 == 0 && v[1]->numel() * 8 == numel &&
                  reinterpret_cast<uintptr_t>(v[1]->data_ptr()) % 16 == 0,
                  "bn mask bits: contiguous uint8 [M, C / 8], C % 128 == 0, 16-byte aligned");
      f.mask = v[1]->data_ptr();
    } else {
      TORCH_CHECK(v[1]->scalar_type() == at::kBFloat16 && v[1]->numel() == numel);
      f.y = v[1]->data_ptr();
    }
  }
  for (int i = 2; i < 7; ++i)
    TORCH_CHECK(v[i].has_value() && v[i]->scalar_type() == at::kFloat && v[i]->is_contiguous() &&
                v[i]->numel() >= (i == 6 ? 2 : 1) * channels, "bn fuse tensor ", i);
  f.mean = v[2]->data_ptr<float>();
  f.rstd = v[3]->data_ptr<float>();
  f.gamma = v[4]->data_ptr<float>();
  f.beta = v[5]->data_ptr<float>();
  f.dsums = v[6]->data_ptr<float>();
  f.relu = relu;
  return f;
}

// The operands of a GEMM: A, B are 2-D bf16 CUDA tensors whose last dimension is contiguous (row pitch = stride(0)).
edl::GemmArgs gemm_operands(const Tensor& A, const Tensor& B, bool a_mn_major, bool b_mn_major) {
  TORCH_CHECK(A.is_cuda() && B.is_cuda() && A.dim() == 2 && B.dim() == 2);
  TORCH_CHECK(A.scalar_type() == at::kBFloat16 && B.scalar_type() == at::kBFloat16);
  TORCH_CHECK(A.stride(1) == 1 && B.stride(1) == 1, "operands need a contiguous last dim");
  edl::GemmArgs g;
  g.A = A.data_ptr();
  g.B = B.data_ptr();
  g.a_mn_major = a_mn_major;
  g.b_mn_major = b_mn_major;
  g.M = a_mn_major ? A.size(1) : A.size(0);
  g.K = a_mn_major ? A.size(0) : A.size(1);
  g.N = b_mn_major ? B.size(1) : B.size(0);
  const int64_t kb = b_mn_major ? B.size(0) : B.size(1);
  TORCH_CHECK(kb == g.K, "K mismatch: ", kb, " vs ", g.K);
  g.lda = A.stride(0);
  g.ldb = B.stride(0);
  TORCH_CHECK(g.lda % 8 == 0 && g.ldb % 8 == 0, "row pitch must be a multiple of 16 bytes");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(g.A) % 16 == 0 && reinterpret_cast<uintptr_t>(g.B) % 16 == 0);
  g.device = A.device().index();
  return g;
}

// D[M,N] = A * B with the operand layouts described in gemm.h (fprop: both K-major; dgrad: B MN-major).
void gemm_bf16(const Tensor& A, const Tensor& B, const Tensor& D, bool a_mn_major, bool b_mn_major,
               const c10::optional<Tensor>& col_scale, const c10::optional<Tensor>& col_shift, bool relu,
               const c10::optional<Tensor>& col_stats, const c10::optional<Tensor>& add_src,
               const c10::optional<std::vector<c10::optional<Tensor>>>& bn, bool bn_relu) {
  TORCH_CHECK(!(a_mn_major && b_mn_major), "both operands MN-major is the weight gradient: use gemm_wgrad_bf16");
  edl::GemmArgs g = gemm_operands(A, B, a_mn_major, b_mn_major);
  TORCH_CHECK(D.scalar_type() == at::kBFloat16);
  TORCH_CHECK(D.dim() == 2 && D.size(0) == g.M && D.size(1) == g.N && D.stride(1) == 1);
  g.D = D.data_ptr();
  g.ldd = D.stride(0);
  TORCH_CHECK(g.ldd % 8 == 0 && reinterpret_cast<uintptr_t>(g.D) % 16 == 0);
  g.col_scale = optp<float>(col_scale);
  g.col_shift = optp<float>(col_shift);
  g.relu = relu;
  g.col_stats = optp<float>(col_stats);
  if (add_src.has_value() && add_src->defined()) {
    TORCH_CHECK(add_src->scalar_type() == at::kBFloat16 && add_src->dim() == 2 && add_src->stride(1) == 1);
    TORCH_CHECK(add_src->size(0) == g.M && add_src->size(1) == g.N);
    g.add_src = add_src->data_ptr();
    g.ld_add = add_src->stride(0);
  }
  if (bn.has_value()) {
    TORCH_CHECK(g.D != nullptr && g.ldd == g.N, "fused BN reduction needs a dense bf16 output");
    g.bn = parse_bn(bn, bn_relu, (int64_t)g.M * g.N, g.N);
  }
  c10::cuda::CUDAGuard guard(A.device());
  const char* err = edl::gemm_bf16(g, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl gemm_bf16 failed: ", err);
}

// D[M,N] = gelu(A * B^T * col_scale + col_shift) (erf form, fp32) on the persistent kernel's GELU epilogue; inference only.
void gemm_bf16_gelu(const Tensor& A, const Tensor& B, const Tensor& D, const c10::optional<Tensor>& col_scale,
                    const c10::optional<Tensor>& col_shift) {
  edl::GemmArgs g = gemm_operands(A, B, false, false);
  TORCH_CHECK(D.scalar_type() == at::kBFloat16);
  TORCH_CHECK(D.dim() == 2 && D.size(0) == g.M && D.size(1) == g.N && D.stride(1) == 1);
  g.D = D.data_ptr();
  g.ldd = D.stride(0);
  TORCH_CHECK(g.ldd % 8 == 0 && reinterpret_cast<uintptr_t>(g.D) % 16 == 0);
  g.col_scale = optp<float>(col_scale);
  g.col_shift = optp<float>(col_shift);
  g.gelu = true;
  c10::cuda::CUDAGuard guard(A.device());
  const char* err = edl::gemm_bf16(g, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl gemm_bf16_gelu failed: ", err);
}

void check_like_d(const Tensor& U, const edl::GemmArgs& g, const char* name) {
  TORCH_CHECK(U.is_cuda() && U.scalar_type() == at::kBFloat16 && U.dim() == 2 && U.size(0) == g.M && U.size(1) == g.N &&
              U.stride(1) == 1 && U.stride(0) % 8 == 0 && reinterpret_cast<uintptr_t>(U.data_ptr()) % 16 == 0, name,
              " must be bf16 [M, N] with 16-byte aligned rows");
}

// Training forward of FFN1: D = gelu(u) and U = u = A * B^T + col_shift (bf16), one persistent GEMM.
void gemm_bf16_gelu_train(const Tensor& A, const Tensor& B, const Tensor& D, const Tensor& U,
                          const c10::optional<Tensor>& col_shift) {
  edl::GemmArgs g = gemm_operands(A, B, false, false);
  check_like_d(D, g, "D");
  check_like_d(U, g, "U");
  g.D = D.data_ptr();
  g.ldd = D.stride(0);
  g.col_shift = optp<float>(col_shift);
  g.gelu = true;
  g.gelu_u = U.data_ptr();
  g.ld_u = U.stride(0);
  c10::cuda::CUDAGuard guard(A.device());
  const char* err = edl::gemm_bf16(g, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl gemm_bf16_gelu_train failed: ", err);
}

// FFN2's dgrad through the GELU: D = (A * B) * gelu'(U), A = dY [M, K], B = W2 [K, N] (MN-major), U = u [M, N].
void gemm_bf16_gelu_grad(const Tensor& A, const Tensor& B, const Tensor& D, const Tensor& U) {
  edl::GemmArgs g = gemm_operands(A, B, false, true);
  check_like_d(D, g, "D");
  check_like_d(U, g, "U");
  g.D = D.data_ptr();
  g.ldd = D.stride(0);
  g.add_src = U.data_ptr();
  g.ld_add = U.stride(0);
  g.gelu_grad = true;
  c10::cuda::CUDAGuard guard(A.device());
  const char* err = edl::gemm_bf16(g, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl gemm_bf16_gelu_grad failed: ", err);
}

// A residual branch with dropout: D = add + Z o (A * B^T + col_shift), Z the mask of `drop` at flat index row * N + col.
void gemm_bf16_residual_dropout(const Tensor& A, const Tensor& B, const Tensor& D, const c10::optional<Tensor>& col_shift,
                                const Tensor& add, const edl::PhiloxArgs& drop) {
  edl::GemmArgs g = gemm_operands(A, B, false, false);
  check_like_d(D, g, "D");
  check_like_d(add, g, "add");
  g.D = D.data_ptr();
  g.ldd = D.stride(0);
  g.col_shift = optp<float>(col_shift);
  g.add_src = add.data_ptr();
  g.ld_add = add.stride(0);
  g.dropout = &drop;
  c10::cuda::CUDAGuard guard(A.device());
  const char* err = edl::gemm_bf16(g, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl gemm_bf16_residual_dropout failed: ", err);
}

// fp32 scratch for the partial tiles of a split reduction (optional: the kernels report it missing or too small)
void set_partials(const c10::optional<Tensor>& partials, float** ptr, int64_t* elems) {
  if (!partials.has_value() || !partials->defined()) return;
  TORCH_CHECK(partials->is_cuda() && partials->scalar_type() == at::kFloat && partials->is_contiguous() &&
              reinterpret_cast<uintptr_t>(partials->data_ptr()) % 16 == 0, "partials: contiguous, aligned fp32");
  *ptr = partials->data_ptr<float>();
  *elems = partials->numel();
}

// Weight gradient of a 1x1 convolution / linear layer: out[N1, N2] (+)= dy[M, N1]^T @ x[M, N2] (bf16, accumulated in
// fp32, one rounding).  split_k > 1 splits the M reduction over CTAs and needs `partials` (see gemm.h GemmArgs).
void gemm_wgrad_bf16(const Tensor& dy, const Tensor& x, Tensor& out, int64_t split_k, bool accumulate,
                     const c10::optional<Tensor>& partials) {
  edl::GemmArgs g = gemm_operands(dy, x, true, true);
  TORCH_CHECK(out.scalar_type() == at::kBFloat16 && out.dim() == 2 && out.size(0) == g.M && out.size(1) <= g.N &&
              out.size(1) > 0 && out.stride(1) == 1, "out must be bf16 [N1, <= N2] with a contiguous last dim");
  if (out.size(1) == g.N) {
    TORCH_CHECK(g.N % 4 == 0 && out.stride(0) % 4 == 0 && reinterpret_cast<uintptr_t>(out.data_ptr()) % 8 == 0,
                "the weight-gradient stores need N2 % 4 == 0 and 8-byte aligned rows");
  } else {
    // a narrower output: only its columns are stored (x's last columns are padding, e.g. the 7x7 stem's im2col)
    g.n_out = (int)out.size(1);
  }
  g.D = out.data_ptr();
  g.ldd = out.stride(0);
  g.split_k = (int)split_k;
  g.accumulate = accumulate;
  set_partials(partials, &g.partials, &g.partials_elems);
  c10::cuda::CUDAGuard guard(dy.device());
  const char* err = edl::gemm_bf16(g, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl gemm_wgrad_bf16 failed: ", err);
}

// Fused "linear -> peer ship": D = A[M,K] * B[N,K]^T (+ bias) TMA-stored straight into a peer GPU's
// buffer at `d_ptr` (row pitch ldd elements); the last CTA releases `flag_ptr` (peer) = seq.
void gemm_bf16_ship(const Tensor& A, const Tensor& B, int64_t d_ptr, int64_t ldd,
                    const c10::optional<Tensor>& col_shift, int64_t flag_ptr,
                    const c10::optional<Tensor>& seq, int64_t seq_imm, const Tensor& done) {
  TORCH_CHECK(A.is_cuda() && B.is_cuda() && A.dim() == 2 && B.dim() == 2);
  TORCH_CHECK(A.scalar_type() == at::kBFloat16 && B.scalar_type() == at::kBFloat16);
  TORCH_CHECK(A.stride(1) == 1 && B.stride(1) == 1 && A.size(1) == B.size(1));
  TORCH_CHECK(done.is_cuda() && done.scalar_type() == at::kInt && done.numel() >= 1);
  edl::GemmArgs g;
  g.A = A.data_ptr();
  g.B = B.data_ptr();
  g.M = A.size(0);
  g.K = A.size(1);
  g.N = B.size(0);
  g.lda = A.stride(0);
  g.ldb = B.stride(0);
  g.D = reinterpret_cast<void*>(d_ptr);
  g.ldd = ldd;
  TORCH_CHECK(g.lda % 8 == 0 && g.ldb % 8 == 0 && g.ldd % 8 == 0 && d_ptr % 16 == 0,
              "row pitches / base must be 16-byte aligned");
  g.col_shift = optp<float>(col_shift);
  g.ship_flag = reinterpret_cast<void*>(flag_ptr);
  g.ship_seq_ptr = seq.has_value() && seq->defined() ? seq->data_ptr() : nullptr;
  g.ship_seq_imm = (uint32_t)seq_imm;
  g.ship_done = done.data_ptr();
  g.device = A.device().index();
  c10::cuda::CUDAGuard guard(A.device());
  const char* err = edl::gemm_bf16(g, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl gemm_bf16_ship failed: ", err);
}

// 3x3 / stride 1 / pad 1 convolution (conv3x3.cu).  x, y: logical NCHW tensors in channels_last memory
// (= NHWC); w: KRSC [Cout, 3, 3, Cin].  dgrad: x is dY [N, Cout, H, W], y is dX [N, Cin, H, W].
void conv3x3(const Tensor& x, const Tensor& w, Tensor& y, bool dgrad, const c10::optional<Tensor>& col_stats,
             const c10::optional<std::vector<c10::optional<Tensor>>>& bn, bool bn_relu) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 4 && y.dim() == 4 && w.dim() == 4);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && y.scalar_type() == at::kBFloat16 &&
              w.scalar_type() == at::kBFloat16);
  TORCH_CHECK(x.is_contiguous(at::MemoryFormat::ChannelsLast) && y.is_contiguous(at::MemoryFormat::ChannelsLast),
              "conv3x3 needs channels_last activations");
  TORCH_CHECK(w.is_contiguous() && w.size(1) == 3 && w.size(2) == 3, "weight must be KRSC [Cout,3,3,Cin]");
  edl::Conv3x3Args a;
  a.X = x.data_ptr();
  a.Wt = w.data_ptr();
  a.Y = y.data_ptr();
  a.N = x.size(0);
  a.H = x.size(2);
  a.W = x.size(3);
  a.Cout = w.size(0);
  a.Cin = w.size(3);
  a.dgrad = dgrad;
  TORCH_CHECK(x.size(1) == (dgrad ? a.Cout : a.Cin) && y.size(1) == (dgrad ? a.Cin : a.Cout));
  TORCH_CHECK(y.size(0) == a.N && y.size(2) == a.H && y.size(3) == a.W);
  a.col_stats = optp<float>(col_stats);
  if (bn.has_value()) {
    TORCH_CHECK(dgrad, "fused BN reduction belongs to the dgrad launch");
    a.bn = parse_bn(bn, bn_relu, y.numel(), y.size(1));
  }
  a.device = x.device().index();
  c10::cuda::CUDAGuard guard(x.device());
  const char* err = edl::conv3x3_bf16(a, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl conv3x3 failed: ", err);
}

// dx [N,Cin,2H,2W] = input gradient of the 3x3 / pad 1 / stride 2 convolution for dy [N,Cout,H,W]; w KRSC [Cout,3,3,Cin]
void conv3x3_dgrad_s2(const Tensor& dy, const Tensor& w, Tensor& dx) {
  TORCH_CHECK(dy.is_cuda() && dy.dim() == 4 && dx.dim() == 4 && w.dim() == 4);
  TORCH_CHECK(dy.scalar_type() == at::kBFloat16 && dx.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16);
  TORCH_CHECK(dy.is_contiguous(at::MemoryFormat::ChannelsLast) && dx.is_contiguous(at::MemoryFormat::ChannelsLast));
  TORCH_CHECK(w.is_contiguous() && w.size(1) == 3 && w.size(2) == 3, "weight must be KRSC [Cout,3,3,Cin]");
  edl::Conv3x3Args a;
  a.X = dy.data_ptr();
  a.Wt = w.data_ptr();
  a.Y = dx.data_ptr();
  a.N = dy.size(0);
  a.H = dy.size(2);
  a.W = dy.size(3);
  a.Cout = w.size(0);
  a.Cin = w.size(3);
  a.dgrad = true;
  TORCH_CHECK(dy.size(1) == a.Cout && dx.size(1) == a.Cin && dx.size(0) == a.N && dx.size(2) == 2 * a.H &&
              dx.size(3) == 2 * a.W, "conv3x3_dgrad_s2: shapes do not belong together");
  a.device = dy.device().index();
  c10::cuda::CUDAGuard guard(dy.device());
  const char* err = edl::conv3x3_dgrad_s2_bf16(a, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl conv3x3_dgrad_s2 failed: ", err);
}
bool conv3x3_dgrad_s2_supported(int64_t n, int64_t ho, int64_t wo, int64_t cin, int64_t cout) {
  return edl::conv3x3_dgrad_s2_supported((int)n, (int)ho, (int)wo, (int)cin, (int)cout);
}

// 1x1 / pad 0 / stride 2 convolution (gemm.h conv1x1_s2_bf16) on the persistent kernel, w [Cout, Cin] (any [Cout, 1, 1, Cin]
// view).  fprop: x [N, Cin, 2H, 2W] -> y [N, Cout, H, W] with col_stats (training) or col_scale / col_shift / relu
// (inference).  dgrad: x is dY [N, Cout, H, W], y is dX [N, Cin, 2H, 2W] (zero-filled, then the even-even pixels).
void conv1x1_s2(const Tensor& x, const Tensor& w, Tensor& y, bool dgrad, const c10::optional<Tensor>& col_stats,
                const c10::optional<Tensor>& col_scale, const c10::optional<Tensor>& col_shift, bool relu) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 4 && y.dim() == 4);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && y.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16);
  TORCH_CHECK(x.is_contiguous(at::MemoryFormat::ChannelsLast) && y.is_contiguous(at::MemoryFormat::ChannelsLast),
              "conv1x1_s2 needs channels_last activations");
  TORCH_CHECK(w.is_contiguous() && w.numel() == w.size(0) * w.size(-1), "weight must be [Cout, Cin] (or [Cout, 1, 1, Cin])");
  const Tensor& in = dgrad ? y : x;      // the convolution's input  [N, Cin, 2H, 2W]
  const Tensor& out = dgrad ? x : y;     // the convolution's output [N, Cout, H, W]
  edl::Conv3x3Args a;
  a.X = x.data_ptr();
  a.Wt = w.data_ptr();
  a.Y = y.data_ptr();
  a.N = out.size(0);
  a.H = out.size(2);
  a.W = out.size(3);
  a.Cout = w.size(0);
  a.Cin = w.size(-1);
  a.dgrad = dgrad;
  a.stride = 2;
  a.ksize = 1;
  TORCH_CHECK(in.size(0) == a.N && in.size(1) == a.Cin && out.size(1) == a.Cout && in.size(2) == 2 * a.H &&
              in.size(3) == 2 * a.W, "conv1x1_s2: x / w / y shapes do not belong together (input 2H x 2W)");
  TORCH_CHECK(!dgrad || (!col_stats.has_value() && !col_scale.has_value() && !col_shift.has_value() && !relu),
              "conv1x1_s2: statistics / epilogue belong to the fprop launch");
  a.col_stats = optp<float>(col_stats);
  a.col_scale = optp<float>(col_scale);
  a.col_shift = optp<float>(col_shift);
  a.relu = relu;
  a.device = x.device().index();
  c10::cuda::CUDAGuard guard(x.device());
  const char* err = edl::conv1x1_s2_bf16(a, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl conv1x1_s2 failed: ", err);
}
bool conv1x1_s2_supported(int64_t n, int64_t ho, int64_t wo, int64_t cin, int64_t cout, bool dgrad) {
  return edl::conv1x1_s2_supported((int)n, (int)ho, (int)wo, (int)cin, (int)cout, dgrad);
}

// dW [Cout, Cin] (+)= weight gradient of the 1x1 / pad 0 / stride 2 convolution: x [N, Cin, 2H, 2W], dy [N, Cout, H, W]
// channels_last; the version-1 weight-gradient kernel with one tap (split_k > 1 needs `partials`: split_k *
// conv3x3_wgrad_tiles(Cin, Cout) / 3 * 128 * 64 floats)
void conv1x1_s2_wgrad(const Tensor& x, const Tensor& dy, Tensor& dw, int64_t split_k, bool accumulate,
                      const c10::optional<Tensor>& partials) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 4 && dy.dim() == 4);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && dy.scalar_type() == at::kBFloat16 && dw.scalar_type() == at::kBFloat16);
  TORCH_CHECK(x.is_contiguous(at::MemoryFormat::ChannelsLast) && dy.is_contiguous(at::MemoryFormat::ChannelsLast),
              "conv1x1_s2_wgrad needs channels_last activations");
  TORCH_CHECK(dw.is_contiguous() && dw.numel() == dw.size(0) * dw.size(-1), "dw must be [Cout, Cin] (or [Cout, 1, 1, Cin])");
  edl::Conv3x3WgradArgs a;
  a.X = x.data_ptr();
  a.dY = dy.data_ptr();
  a.dW = dw.data_ptr();
  a.N = x.size(0);
  a.H = dy.size(2);
  a.W = dy.size(3);
  a.Cin = x.size(1);
  a.Cout = dy.size(1);
  a.stride = 2;
  a.ksize = 1;
  TORCH_CHECK(dy.size(0) == a.N && x.size(2) == 2 * a.H && x.size(3) == 2 * a.W && dw.size(0) == a.Cout &&
              dw.size(-1) == a.Cin, "conv1x1_s2_wgrad: x / dy / dw shapes do not belong together");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(a.dW) % 8 == 0, "dw window must be 8-byte aligned");
  a.split_k = (int)split_k;
  a.accumulate = accumulate;
  set_partials(partials, &a.partials, &a.partials_elems);
  a.device = x.device().index();
  c10::cuda::CUDAGuard guard(x.device());
  const char* err = edl::conv3x3_wgrad_bf16(a, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl conv1x1_s2_wgrad failed: ", err);
}

inline bool aligned16(const Tensor& t) { return reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0; }

// The operand checks shared by every fp8 GEMM entry: A [M, K] and B [N, K] hold e4m3 bytes, D is [M, N] (bf16, or e4m3
// bytes for the GELU epilogue), all on one CUDA device with 16-byte aligned bases and rows, K % 16 == 0; col_scale /
// col_shift (optional) are contiguous fp32 [N] on that device.
void fp8_gemm_checks(const Tensor& A, const Tensor& B, const Tensor& D, const c10::optional<Tensor>& col_scale,
                     const c10::optional<Tensor>& col_shift, bool q_out) {
  TORCH_CHECK(A.is_cuda() && B.is_cuda() && D.is_cuda() && A.dim() == 2 && B.dim() == 2 && D.dim() == 2,
              "A, B and D must be 2-D CUDA tensors");
  TORCH_CHECK(A.device() == B.device() && A.device() == D.device(), "A, B and D on different devices");
  TORCH_CHECK(A.element_size() == 1 && B.element_size() == 1, "A and B hold e4m3 bytes");
  if (q_out) {
    TORCH_CHECK(D.element_size() == 1, "the GELU e4m3 epilogue writes e4m3 bytes");
  } else {
    TORCH_CHECK(D.scalar_type() == at::kBFloat16, "D must be bf16");
  }
  TORCH_CHECK(A.stride(1) == 1 && B.stride(1) == 1 && D.stride(1) == 1, "operands need a contiguous last dim");
  TORCH_CHECK(A.size(1) == B.size(1), "K mismatch: ", A.size(1), " vs ", B.size(1));
  TORCH_CHECK(D.size(0) == A.size(0) && D.size(1) == B.size(0), "D must be [M, N]");
  TORCH_CHECK(A.size(1) % 16 == 0 && A.stride(0) % 16 == 0 && B.stride(0) % 16 == 0 &&
              D.stride(0) % (q_out ? 16 : 8) == 0, "fp8 GEMM needs 16-byte aligned rows");
  TORCH_CHECK(aligned16(A) && aligned16(B) && aligned16(D), "A, B and D must be 16-byte aligned");
  for (const auto* t : {&col_scale, &col_shift})
    if (t->has_value() && (*t)->defined())
      TORCH_CHECK((*t)->is_cuda() && (*t)->device() == A.device() && (*t)->scalar_type() == at::kFloat &&
                  (*t)->is_contiguous() && (*t)->numel() == B.size(0),
                  "col_scale / col_shift must be contiguous fp32 [N] on the operands' device");
}

// D bf16 [M,N] = relu?((A8[M,K] * B8[N,K]^T) * col_scale + col_shift); A8/B8 are e4m3 bytes (uint8 / float8 tensors)
void gemm_fp8(const Tensor& A, const Tensor& B, Tensor& D, const c10::optional<Tensor>& col_scale,
              const c10::optional<Tensor>& col_shift, bool relu) {
  fp8_gemm_checks(A, B, D, col_scale, col_shift, false);
  edl::GemmFp8Args g;
  g.A = A.data_ptr();
  g.B = B.data_ptr();
  g.D = D.data_ptr();
  g.M = A.size(0);
  g.K = A.size(1);
  g.N = B.size(0);
  g.lda = A.stride(0);
  g.ldb = B.stride(0);
  g.ldd = D.stride(0);
  g.col_scale = optp<float>(col_scale);
  g.col_shift = optp<float>(col_shift);
  g.relu = relu;
  g.device = A.device().index();
  c10::cuda::CUDAGuard guard(A.device());
  const char* err = edl::gemm_fp8(g, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl gemm_fp8 failed: ", err);
}

// q = sat(x / scale) as e4m3 bytes, x bf16 (read as 16-byte vectors), q written 8 bytes at a time; scale and the
// optional running max|x| `amax` are fp32 device scalars the kernel dereferences
void quantize_e4m3(const Tensor& x, Tensor& q, const Tensor& scale, const c10::optional<Tensor>& amax) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16 && x.is_contiguous(), "x must be a contiguous bf16 CUDA tensor");
  TORCH_CHECK(aligned16(x), "x must be 16-byte aligned");
  TORCH_CHECK(q.is_cuda() && q.device() == x.device() && q.element_size() == 1 && q.is_contiguous() &&
              q.numel() == x.numel(), "q must be a contiguous 1-byte tensor of x's size on x's device");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(q.data_ptr()) % 8 == 0, "q must be 8-byte aligned");
  TORCH_CHECK(scale.is_cuda() && scale.device() == x.device() && scale.scalar_type() == at::kFloat && scale.numel() >= 1,
              "scale must be an fp32 tensor on x's device");
  if (amax.has_value() && amax->defined())
    TORCH_CHECK(amax->is_cuda() && amax->device() == x.device() && amax->scalar_type() == at::kFloat &&
                amax->numel() >= 1, "amax must be an fp32 tensor on x's device");
  c10::cuda::CUDAGuard guard(x.device());
  edl::quantize_e4m3(x.data_ptr(), q.data_ptr(), x.numel(), scale.data_ptr<float>(), optp<float>(amax),
                     at::cuda::getCurrentCUDAStream().stream());
}

// q [M, K] e4m3 bytes (contiguous), sa fp32 [ceil(K/128), M] = per-row, per-128-element-block scales of x [M, K]
void quantize_e4m3_blocks(const Tensor& x, Tensor& q, Tensor& sa) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 2 && x.scalar_type() == at::kBFloat16, "x must be a 2-D bf16 CUDA tensor");
  TORCH_CHECK(x.stride(1) == 1, "x needs a contiguous last dim");
  const int64_t M = x.size(0), K = x.size(1), kb = (K + 127) / 128;
  TORCH_CHECK(M > 0 && K > 0 && K % 8 == 0, "block quantiser needs K % 8 == 0, got K = ", K);
  TORCH_CHECK(x.stride(0) % 8 == 0 && reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0,
              "x rows must be 16-byte aligned");
  TORCH_CHECK(q.is_cuda() && q.element_size() == 1 && q.is_contiguous() && q.dim() == 2 && q.size(0) == M &&
              q.size(1) == K, "q must be a contiguous 1-byte [M, K] tensor");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(q.data_ptr()) % 8 == 0, "q must be 8-byte aligned");
  TORCH_CHECK(sa.is_cuda() && sa.scalar_type() == at::kFloat && sa.is_contiguous() && sa.dim() == 2 &&
              sa.size(0) == kb && sa.size(1) == M, "sa must be contiguous fp32 [ceil(K/128), M]");
  TORCH_CHECK(x.device() == q.device() && x.device() == sa.device(), "tensors on different devices");
  c10::cuda::CUDAGuard guard(x.device());
  const char* err = edl::quantize_e4m3_blocks(x.data_ptr(), x.stride(0), q.data_ptr(), sa.data_ptr<float>(), (int)M,
                                              (int)K, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl quantize_e4m3_blocks failed: ", err);
}

// The checks and arguments shared by the block-scaled entries (D: bf16, or e4m3 bytes for the GELU epilogue)
edl::GemmFp8Args blockscaled_args(const Tensor& A, const Tensor& sa, const Tensor& B, const Tensor& sb, const Tensor& D,
                                  const c10::optional<Tensor>& col_scale, const c10::optional<Tensor>& col_shift,
                                  bool relu, bool q_out) {
  fp8_gemm_checks(A, B, D, col_scale, col_shift, q_out);
  const int64_t M = A.size(0), N = B.size(0), K = A.size(1), kb = (K + 127) / 128;
  TORCH_CHECK(sa.is_cuda() && sa.device() == A.device() && sa.scalar_type() == at::kFloat && sa.is_contiguous() &&
              sa.dim() == 2 && sa.size(0) == kb && sa.size(1) == M, "sa must be contiguous fp32 [ceil(K/128), M]");
  TORCH_CHECK(sb.is_cuda() && sb.device() == A.device() && sb.scalar_type() == at::kFloat && sb.is_contiguous() &&
              sb.dim() == 2 && sb.size(0) == (N + 127) / 128 && sb.size(1) == kb,
              "sb must be contiguous fp32 [ceil(N/128), ceil(K/128)]");
  edl::GemmFp8Args g;
  g.A = A.data_ptr();
  g.B = B.data_ptr();
  g.D = D.data_ptr();
  g.M = M;
  g.K = K;
  g.N = N;
  g.lda = A.stride(0);
  g.ldb = B.stride(0);
  g.ldd = D.stride(0);
  g.col_scale = optp<float>(col_scale);
  g.col_shift = optp<float>(col_shift);
  g.relu = relu;
  g.a_scales = sa.data_ptr<float>();
  g.b_scales = sb.data_ptr<float>();
  g.device = A.device().index();
  return g;
}

// D bf16 [M,N] = relu?((sum_b (A8_b * B8_b^T) * sa[b, m] * sb[n / 128, b]) * col_scale + col_shift (+ add))
void gemm_fp8_blockscaled(const Tensor& A, const Tensor& sa, const Tensor& B, const Tensor& sb, Tensor& D,
                          const c10::optional<Tensor>& col_scale, const c10::optional<Tensor>& col_shift, bool relu,
                          const c10::optional<Tensor>& add) {
  edl::GemmFp8Args g = blockscaled_args(A, sa, B, sb, D, col_scale, col_shift, relu, false);
  if (add.has_value() && add->defined()) {
    TORCH_CHECK(add->is_cuda() && add->device() == D.device() && add->scalar_type() == at::kBFloat16 &&
                add->dim() == 2 && add->size(0) == g.M && add->size(1) == g.N && add->stride(1) == 1,
                "add must be a bf16 [M, N] CUDA tensor with a contiguous last dim");
    TORCH_CHECK(g.N % 8 == 0 && add->stride(0) % 8 == 0 && reinterpret_cast<uintptr_t>(add->data_ptr()) % 16 == 0,
                "add needs 16-byte aligned rows");
    g.add = add->data_ptr();
    g.ld_add = add->stride(0);
  }
  c10::cuda::CUDAGuard guard(A.device());
  const char* err = edl::gemm_fp8_blockscaled(g, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl gemm_fp8_blockscaled failed: ", err);
}

// Q e4m3 [M,N], sa_out fp32 [ceil(N/128), M]: block quantisation of bf16(gelu(sum_b (A8_b * B8_b^T) * sa * sb + bias))
void gemm_fp8_blockscaled_gelu_e4m3(const Tensor& A, const Tensor& sa, const Tensor& B, const Tensor& sb, Tensor& Q,
                                    Tensor& sa_out, const c10::optional<Tensor>& bias) {
  edl::GemmFp8Args g = blockscaled_args(A, sa, B, sb, Q, c10::nullopt, bias, false, true);
  TORCH_CHECK(g.N % 16 == 0, "the GELU e4m3 epilogue needs N % 16 == 0, got N = ", g.N);
  TORCH_CHECK(sa_out.is_cuda() && sa_out.device() == Q.device() && sa_out.scalar_type() == at::kFloat &&
              sa_out.is_contiguous() && sa_out.dim() == 2 && sa_out.size(0) == (g.N + 127) / 128 &&
              sa_out.size(1) == g.M, "sa_out must be contiguous fp32 [ceil(N/128), M]");
  g.a_scales_out = sa_out.data_ptr<float>();
  c10::cuda::CUDAGuard guard(A.device());
  const char* err = edl::gemm_fp8_blockscaled_gelu_e4m3(g, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl gemm_fp8_blockscaled_gelu_e4m3 failed: ", err);
}

bool conv3x3_supported(int64_t n, int64_t h, int64_t w, int64_t cin, int64_t cout, bool dgrad, int64_t groups) {
  return edl::conv3x3_supported((int)n, (int)h, (int)w, (int)cin, (int)cout, dgrad, (int)groups);
}

// dW (+)= wgrad of the 3x3 / stride 1 / pad 1 conv.  x [N,Cin,H,W], dy [N,Cout,H,W] channels_last; dw KRSC
// [Cout,3,3,Cin] bf16 contiguous; split_k > 1 needs `partials` (see gemm.h Conv3x3WgradArgs).
void conv3x3_wgrad(const Tensor& x, const Tensor& dy, Tensor& dw, int64_t split_k, bool accumulate,
                   const c10::optional<Tensor>& partials) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 4 && dy.dim() == 4 && dw.dim() == 4);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && dy.scalar_type() == at::kBFloat16 && dw.scalar_type() == at::kBFloat16);
  TORCH_CHECK(x.is_contiguous(at::MemoryFormat::ChannelsLast) && dy.is_contiguous(at::MemoryFormat::ChannelsLast),
              "conv3x3_wgrad needs channels_last activations");
  TORCH_CHECK(dw.is_contiguous() && dw.size(1) == 3 && dw.size(2) == 3, "dw must be KRSC [Cout,3,3,Cin]");
  edl::Conv3x3WgradArgs a;
  a.X = x.data_ptr();
  a.dY = dy.data_ptr();
  a.dW = dw.data_ptr();
  a.N = x.size(0);
  a.H = dy.size(2);
  a.W = dy.size(3);
  a.Cin = x.size(1);
  a.Cout = dy.size(1);
  // stride 1: x and dy have the same size; stride 2: x is twice as large in both directions
  a.stride = (x.size(2) == 2 * a.H && x.size(3) == 2 * a.W && a.H != x.size(2)) ? 2 : 1;
  TORCH_CHECK(dy.size(0) == a.N && x.size(2) == a.stride * a.H && x.size(3) == a.stride * a.W &&
              dw.size(0) == a.Cout && dw.size(3) == a.Cin, "conv3x3_wgrad: x / dy / dw shapes do not belong together");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(a.dW) % 8 == 0, "dw window must be 8-byte aligned");
  a.split_k = (int)split_k;
  a.accumulate = accumulate;
  set_partials(partials, &a.partials, &a.partials_elems);
  a.device = x.device().index();
  c10::cuda::CUDAGuard guard(x.device());
  const char* err = edl::conv3x3_wgrad_bf16(a, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl conv3x3_wgrad failed: ", err);
}

// 3x3 / pad 1 / STRIDE 2 fprop (dense or grouped) on the persistent kernel: x [N, Cin, 2H, 2W], y [N, Cout, H, W]
// channels_last.  Training use: col_stats (BN statistics of y); inference use: col_scale / col_shift / relu.
void conv3x3_s2(const Tensor& x, const Tensor& w, Tensor& y, const c10::optional<Tensor>& col_stats,
                const c10::optional<Tensor>& col_scale, const c10::optional<Tensor>& col_shift, bool relu,
                int64_t groups) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 4 && y.dim() == 4 && w.dim() == 4);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && y.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16);
  TORCH_CHECK(x.is_contiguous(at::MemoryFormat::ChannelsLast) && y.is_contiguous(at::MemoryFormat::ChannelsLast));
  TORCH_CHECK(w.is_contiguous() && w.size(1) == 3 && w.size(2) == 3);
  edl::Conv3x3Args a;
  a.X = x.data_ptr();
  a.Wt = w.data_ptr();
  a.Y = y.data_ptr();
  a.N = y.size(0);
  a.H = y.size(2);
  a.W = y.size(3);
  a.Cin = x.size(1);
  a.Cout = w.size(0);
  a.groups = (int)groups;
  a.stride = 2;
  TORCH_CHECK(x.size(0) == a.N && x.size(2) == 2 * a.H && x.size(3) == 2 * a.W, "stride-2 conv needs an even input: x is 2H x 2W");
  TORCH_CHECK(w.size(3) * groups == a.Cin && y.size(1) == a.Cout);
  a.col_stats = optp<float>(col_stats);
  a.col_scale = optp<float>(col_scale);
  a.col_shift = optp<float>(col_shift);
  a.relu = relu;
  a.device = x.device().index();
  c10::cuda::CUDAGuard guard(x.device());
  const char* err = edl::conv3x3_bf16(a, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl conv3x3_s2 failed: ", err);
}

std::vector<int64_t> conv3x3_wgrad_plan(int64_t n, int64_t h, int64_t w) {
  int bh = 0, nb = 0, kb = 0;
  edl::conv3x3_wgrad_plan((int)n, (int)h, (int)w, &bh, &nb, &kb);
  // box width: W for version 1; for version 2 the box starts at column -1 and spans kb / (bh * nb) >= W + 1 columns
  const int wb = (bh > 0 && nb > 0) ? kb / (bh * nb) : 0;
  return {bh, nb, kb, wb};
}

bool conv3x3_wgrad_supported(int64_t n, int64_t h, int64_t w, int64_t cin, int64_t cout) {
  return edl::conv3x3_wgrad_supported((int)n, (int)h, (int)w, (int)cin, (int)cout);
}
bool conv3x3_wgrad_s2_supported(int64_t n, int64_t ho, int64_t wo, int64_t cin, int64_t cout) {
  return edl::conv3x3_wgrad_s2_supported((int)n, (int)ho, (int)wo, (int)cin, (int)cout);
}

// inference 3x3 conv (optionally grouped) with the folded-BN scale / shift / ReLU epilogue
void conv3x3_infer(const Tensor& x, const Tensor& w, Tensor& y, const c10::optional<Tensor>& col_scale,
                   const c10::optional<Tensor>& col_shift, bool relu, int64_t groups) {
  TORCH_CHECK(x.is_cuda() && x.dim() == 4 && y.dim() == 4 && w.dim() == 4);
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && y.scalar_type() == at::kBFloat16 && w.scalar_type() == at::kBFloat16);
  TORCH_CHECK(x.is_contiguous(at::MemoryFormat::ChannelsLast) && y.is_contiguous(at::MemoryFormat::ChannelsLast));
  TORCH_CHECK(w.is_contiguous() && w.size(1) == 3 && w.size(2) == 3);
  edl::Conv3x3Args a;
  a.X = x.data_ptr();
  a.Wt = w.data_ptr();
  a.Y = y.data_ptr();
  a.N = x.size(0);
  a.H = x.size(2);
  a.W = x.size(3);
  a.Cin = x.size(1);
  a.Cout = w.size(0);
  a.groups = (int)groups;
  TORCH_CHECK(w.size(3) * groups == a.Cin && y.size(1) == a.Cout && y.size(0) == a.N && y.size(2) == a.H && y.size(3) == a.W);
  a.col_scale = optp<float>(col_scale);
  a.col_shift = optp<float>(col_shift);
  a.relu = relu;
  a.device = x.device().index();
  c10::cuda::CUDAGuard guard(x.device());
  const char* err = edl::conv3x3_bf16(a, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl conv3x3_infer failed: ", err);
}
}  // namespace

void register_gemm_bindings(pybind11::module_& m) {
  m.def("gemm_bf16", &gemm_bf16);
  m.def("gemm_bf16_gelu", &gemm_bf16_gelu);
  m.def("gemm_bf16_gelu_train", &gemm_bf16_gelu_train);
  m.def("gemm_bf16_gelu_grad", &gemm_bf16_gelu_grad);
  m.def("gemm_bf16_residual_dropout", &gemm_bf16_residual_dropout);
  m.def("gemm_wgrad_bf16", &gemm_wgrad_bf16);
  m.def("conv3x3", &conv3x3);
  m.def("set_persistent_gemm", &edl::set_persistent_gemm);
  m.def("get_bnr_mode", &edl::get_bnr_mode);
  m.def("persistent_gemm_enabled", &edl::persistent_gemm_enabled);
  m.def("gemm_fp8", &gemm_fp8);
  m.def("quantize_e4m3", &quantize_e4m3);
  m.def("gemm_fp8_blockscaled", &gemm_fp8_blockscaled, pybind11::arg("A"), pybind11::arg("sa"), pybind11::arg("B"), pybind11::arg("sb"),
        pybind11::arg("D"), pybind11::arg("col_scale"), pybind11::arg("col_shift"), pybind11::arg("relu"), pybind11::arg("add") = pybind11::none());
  m.def("gemm_fp8_blockscaled_gelu_e4m3", &gemm_fp8_blockscaled_gelu_e4m3);
  m.def("quantize_e4m3_blocks", &quantize_e4m3_blocks);
  m.def("conv3x3_supported", &conv3x3_supported);
  m.def("conv3x3_infer", &conv3x3_infer);
  m.def("gemm_bf16_ship", &gemm_bf16_ship);
  m.def("conv3x3_dgrad_s2", &conv3x3_dgrad_s2);
  m.def("conv3x3_dgrad_s2_supported", &conv3x3_dgrad_s2_supported);
  m.def("conv3x3_wgrad", &conv3x3_wgrad);
  m.def("conv3x3_wgrad_supported", &conv3x3_wgrad_supported);
  m.def("conv3x3_wgrad_s2_supported", &conv3x3_wgrad_s2_supported);
  m.def("conv3x3_wgrad_s2_kblocks", &edl::conv3x3_wgrad_s2_kblocks);
  m.def("conv3x3_wgrad_tiles", &edl::conv3x3_wgrad_tiles);
  m.def("conv3x3_wgrad_kblocks", &edl::conv3x3_wgrad_kblocks);
  m.def("conv3x3_wgrad_ctas", &edl::conv3x3_wgrad_ctas);
  m.def("set_wide_gemm_tiles", &edl::set_wide_gemm_tiles);
  m.def("set_persist_trace", [](c10::optional<Tensor> t) {
    if (!t.has_value()) { edl::set_persist_trace(nullptr); return; }
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kLong && t->numel() >= 3 * 16 * 8 && t->is_contiguous(),
                "trace buffer: contiguous CUDA int64 tensor with at least 384 elements");
    edl::set_persist_trace(reinterpret_cast<long long*>(t->data_ptr<int64_t>()));
  });
  m.def("set_epilogue_warps", &edl::set_epilogue_warps);
  m.def("conv3x3_halo_plan", [](int64_t n, int64_t h, int64_t w) -> std::vector<int64_t> {
    int bh = 0, bn = 0, th = 0, ti = 0;
    if (!edl::conv3x3_halo_plan((int)n, (int)h, (int)w, &bh, &bn, &th, &ti)) return {};
    return {bh, bn, th, ti};
  });
  m.def("set_conv_halo", &edl::set_conv_halo);
  m.def("get_conv_halo", &edl::get_conv_halo);
  m.def("set_conv_resident_weights", &edl::set_conv_resident_weights);
  m.def("set_wgrad3_version", &edl::set_wgrad3_version);
  m.def("get_wgrad3_version", &edl::get_wgrad3_version);
  m.def("conv3x3_wgrad_plan", &conv3x3_wgrad_plan);
  m.def("conv3x3_s2", &conv3x3_s2);
  m.def("conv1x1_s2", &conv1x1_s2);
  m.def("conv1x1_s2_supported", &conv1x1_s2_supported);
  m.def("conv1x1_s2_wgrad", &conv1x1_s2_wgrad);
}
