// torch bindings for the Transformer encoder kernels (attention.cu, attention_bwd.cu, layernorm.cu and its quantising
// variants, dropout.cu).
#include <ATen/cuda/CUDAContext.h>
#include <ATen/cuda/CUDAGeneratorImpl.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include <cmath>
#include <mutex>

#include "kernels.h"

namespace {
using torch::Tensor;

// One dropout site: 4 offset units of the default CUDA generator of `device` (graph-safe: under capture the kernels read
// the seed and offset through the generator's device pointers), threshold floor(p * 2^32) and scale fp32(1 / (1 - p)).
edl::PhiloxArgs dropout_draw(int64_t device, double p) {
  TORCH_CHECK(p > 0.0 && p < 1.0, "dropout_draw: 0 < p < 1");
  auto gen = at::get_generator_or_default<at::CUDAGeneratorImpl>(
      std::nullopt, at::cuda::detail::getDefaultCUDAGenerator((c10::DeviceIndex)device));
  at::PhiloxCudaState st;
  {
    std::lock_guard<std::mutex> lock(gen->mutex_);
    st = gen->philox_cuda_state(4);
  }
  edl::PhiloxArgs a;
  if (st.captured_) {
    a.seed_ptr = st.seed_.ptr;
    a.offset_ptr = st.offset_.ptr;
    a.offset_intragraph = st.offset_intragraph_;
  } else {
    a.seed = st.seed_.val;
    a.offset = st.offset_.val;
  }
  a.threshold = (uint32_t)std::floor(p * 4294967296.0);
  a.scale = (float)(1.0 / (1.0 - p));
  return a;
}

// y = Z o x, x / y bf16 CUDA tensors of one size (contiguous)
void dropout_fwd(const Tensor& x, Tensor& y, const edl::PhiloxArgs& drop) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kBFloat16 && x.is_contiguous() && y.is_cuda() &&
              y.scalar_type() == at::kBFloat16 && y.is_contiguous() && y.numel() == x.numel() &&
              y.device() == x.device(), "dropout: x, y contiguous bf16 CUDA tensors of one size");
  c10::cuda::CUDAGuard guard(x.device());
  edl::dropout_apply(x.data_ptr(), y.data_ptr(), x.numel(), drop, at::cuda::getCurrentCUDAStream().stream());
}

void check_bf16_2d(const Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.dim() == 2 && t.scalar_type() == at::kBFloat16 && t.is_contiguous(), name,
              " must be a contiguous 2-D bf16 CUDA tensor");
}

// The head dim D of a qkv [rows, 3 * H * D]: 64 or 32, the widths the attention kernels take
int64_t head_dim(const Tensor& qkv, int64_t H) {
  TORCH_CHECK(H >= 1, "attention: H >= 1 heads");
  const int64_t D = qkv.size(1) / (3 * H);
  TORCH_CHECK(qkv.size(1) == 3 * H * D && (D == 64 || D == 32),
              "attention: qkv must be [rows, 3 * H * D] with head dim D = 64 or 32, got width ", qkv.size(1),
              " for H = ", H);
  return D;
}

// qkv [B * L, 3 * H * D], mask uint8 [B, L] or None, out [B * L, H * D]; D = 64 or 32
void attention_fwd(const Tensor& qkv, const c10::optional<Tensor>& mask, Tensor& out, int64_t B, int64_t L, int64_t H,
                   const c10::optional<Tensor>& lse, const edl::PhiloxArgs* drop) {
  check_bf16_2d(qkv, "qkv");
  check_bf16_2d(out, "out");
  const int64_t D = head_dim(qkv, H);
  TORCH_CHECK(qkv.size(0) == B * L, "qkv must be [B * L, 3 * H * D]");
  TORCH_CHECK(out.size(0) == B * L && out.size(1) == H * D, "out must be [B * L, H * D]");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(qkv.data_ptr()) % 16 == 0 && reinterpret_cast<uintptr_t>(out.data_ptr()) % 16 == 0);
  const uint8_t* mp = nullptr;
  if (mask.has_value() && mask->defined()) {
    TORCH_CHECK(mask->is_cuda() && mask->scalar_type() == at::kByte && mask->is_contiguous() && mask->numel() == B * L,
                "mask must be a contiguous uint8 [B, L] CUDA tensor");
    mp = mask->data_ptr<uint8_t>();
  }
  float* lp = nullptr;
  if (lse.has_value() && lse->defined()) {
    TORCH_CHECK(lse->is_cuda() && lse->scalar_type() == at::kFloat && lse->is_contiguous() && lse->numel() == B * H * L,
                "lse must be a contiguous fp32 [B, H, L] CUDA tensor");
    lp = lse->data_ptr<float>();
  }
  c10::cuda::CUDAGuard guard(qkv.device());
  const char* err = edl::attention_fwd(qkv.data_ptr(), mp, out.data_ptr(), (int)B, (int)L, (int)H, (int)D,
                                       at::cuda::getCurrentCUDAStream().stream(), lp, drop);
  TORCH_CHECK(err == nullptr, "edl attention_fwd failed: ", err);
}

// dqkv [B * L, 3 * H * D] from qkv, the forward's out and lse [B, H, L], dout [B * L, H * D]; delta fp32 [B, H, L]
void attention_bwd(const Tensor& qkv, const c10::optional<Tensor>& mask, const Tensor& out, const Tensor& lse,
                   const Tensor& dout, Tensor& dqkv, Tensor& delta, int64_t B, int64_t L, int64_t H,
                   const edl::PhiloxArgs* drop) {
  for (const Tensor* t : {&qkv, &out, &dout, static_cast<const Tensor*>(&dqkv)}) check_bf16_2d(*t, "attention_bwd operand");
  const int64_t D = head_dim(qkv, H);
  TORCH_CHECK(qkv.size(0) == B * L && dqkv.sizes() == qkv.sizes(), "qkv / dqkv must be [B * L, 3 * H * D]");
  TORCH_CHECK(out.size(0) == B * L && out.size(1) == H * D && dout.sizes() == out.sizes(), "out / dout: [B * L, H * D]");
  for (const Tensor* t : {&lse, static_cast<const Tensor*>(&delta)})
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kFloat && t->is_contiguous() && t->numel() == B * H * L,
                "lse / delta must be contiguous fp32 [B, H, L] CUDA tensors");
  for (const Tensor* t : {&qkv, &out, &dout, static_cast<const Tensor*>(&dqkv)})
    TORCH_CHECK(reinterpret_cast<uintptr_t>(t->data_ptr()) % 16 == 0 && t->device() == qkv.device());
  const uint8_t* mp = nullptr;
  if (mask.has_value() && mask->defined()) {
    TORCH_CHECK(mask->is_cuda() && mask->scalar_type() == at::kByte && mask->is_contiguous() && mask->numel() == B * L,
                "mask must be a contiguous uint8 [B, L] CUDA tensor");
    mp = mask->data_ptr<uint8_t>();
  }
  c10::cuda::CUDAGuard guard(qkv.device());
  const char* err = edl::attention_bwd(qkv.data_ptr(), mp, out.data_ptr(), lse.data_ptr<float>(), dout.data_ptr(),
                                       dqkv.data_ptr(), delta.data_ptr<float>(), (int)B, (int)L, (int)H, (int)D,
                                       at::cuda::getCurrentCUDAStream().stream(), drop);
  TORCH_CHECK(err == nullptr, "edl attention_bwd failed: ", err);
}

// cu_seqlens int32 [B + 1] and key_mask uint8 [T] or None of a packed batch of T rows; returns B
int64_t check_varlen(const Tensor& cu_seqlens, const c10::optional<Tensor>& key_mask, int64_t T, const uint8_t** mp) {
  const int64_t B = cu_seqlens.numel() - 1;
  TORCH_CHECK(cu_seqlens.is_cuda() && cu_seqlens.scalar_type() == at::kInt && cu_seqlens.dim() == 1 &&
              cu_seqlens.is_contiguous() && B >= 1, "cu_seqlens must be a contiguous int32 [B + 1] CUDA tensor");
  TORCH_CHECK(T < (int64_t{1} << 31) && B <= 65535, "attention_varlen: T < 2^31 rows, B <= 65535 sequences");
  *mp = nullptr;
  if (key_mask.has_value() && key_mask->defined()) {
    TORCH_CHECK(key_mask->is_cuda() && key_mask->scalar_type() == at::kByte && key_mask->is_contiguous() &&
                key_mask->numel() == T, "key_mask must be a contiguous uint8 [T] CUDA tensor");
    *mp = key_mask->data_ptr<uint8_t>();
  }
  return B;
}

// qkv [T, 3 * H * D], cu_seqlens int32 [B + 1], key_mask uint8 [T] or None, out [T, H * D], maps uint8 [B * 256];
// training: lse fp32 [H, T] (and drop, with lse) or None
void attention_varlen_fwd(const Tensor& qkv, const Tensor& cu_seqlens, const c10::optional<Tensor>& key_mask,
                          Tensor& out, Tensor& maps, int64_t max_len, int64_t H, const c10::optional<Tensor>& lse,
                          const edl::PhiloxArgs* drop) {
  check_bf16_2d(qkv, "qkv");
  check_bf16_2d(out, "out");
  const int64_t T = qkv.size(0);
  const int64_t D = head_dim(qkv, H);
  TORCH_CHECK(out.size(0) == T && out.size(1) == H * D, "out must be [T, H * D]");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(qkv.data_ptr()) % 16 == 0 && reinterpret_cast<uintptr_t>(out.data_ptr()) % 16 == 0);
  const uint8_t* mp;
  const int64_t B = check_varlen(cu_seqlens, key_mask, T, &mp);
  TORCH_CHECK(maps.is_cuda() && maps.scalar_type() == at::kByte && maps.is_contiguous() && maps.numel() >= B * 256 &&
              reinterpret_cast<uintptr_t>(maps.data_ptr()) % 64 == 0, "maps: 64-byte aligned uint8 [B * 256] workspace");
  float* lp = nullptr;
  if (lse.has_value() && lse->defined()) {
    TORCH_CHECK(lse->is_cuda() && lse->scalar_type() == at::kFloat && lse->is_contiguous() && lse->numel() == H * T &&
                lse->device() == qkv.device(), "lse must be a contiguous fp32 [H, T] CUDA tensor");
    lp = lse->data_ptr<float>();
  }
  c10::cuda::CUDAGuard guard(qkv.device());
  const char* err = edl::attention_varlen_fwd(qkv.data_ptr(), cu_seqlens.data_ptr<int>(), mp, out.data_ptr(),
                                              maps.data_ptr(), (int)T, (int)B, (int)max_len, (int)H, (int)D,
                                              at::cuda::getCurrentCUDAStream().stream(), lp, drop);
  TORCH_CHECK(err == nullptr, "edl attention_varlen_fwd failed: ", err);
}

// dqkv [T, 3 * H * D] (the rows of every sequence) from qkv, the packed forward's out and lse [H, T], dout [T, H * D];
// delta fp32 [H, T]
void attention_varlen_bwd(const Tensor& qkv, const Tensor& cu_seqlens, const c10::optional<Tensor>& key_mask,
                          const Tensor& out, const Tensor& lse, const Tensor& dout, Tensor& dqkv, Tensor& delta,
                          int64_t max_len, int64_t H, const edl::PhiloxArgs* drop) {
  for (const Tensor* t : {&qkv, &out, &dout, static_cast<const Tensor*>(&dqkv)})
    check_bf16_2d(*t, "attention_varlen_bwd operand");
  const int64_t T = qkv.size(0);
  const int64_t D = head_dim(qkv, H);
  TORCH_CHECK(dqkv.sizes() == qkv.sizes(), "qkv / dqkv must be [T, 3 * H * D]");
  TORCH_CHECK(out.size(0) == T && out.size(1) == H * D && dout.sizes() == out.sizes(), "out / dout: [T, H * D]");
  for (const Tensor* t : {&lse, static_cast<const Tensor*>(&delta)})
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kFloat && t->is_contiguous() && t->numel() == H * T &&
                t->device() == qkv.device(), "lse / delta must be contiguous fp32 [H, T] CUDA tensors");
  for (const Tensor* t : {&qkv, &out, &dout, static_cast<const Tensor*>(&dqkv)})
    TORCH_CHECK(reinterpret_cast<uintptr_t>(t->data_ptr()) % 16 == 0 && t->device() == qkv.device());
  const uint8_t* mp;
  const int64_t B = check_varlen(cu_seqlens, key_mask, T, &mp);
  c10::cuda::CUDAGuard guard(qkv.device());
  const char* err = edl::attention_varlen_bwd(qkv.data_ptr(), cu_seqlens.data_ptr<int>(), mp, out.data_ptr(),
                                              lse.data_ptr<float>(), dout.data_ptr(), dqkv.data_ptr(),
                                              delta.data_ptr<float>(), (int)T, (int)B, (int)max_len, (int)H, (int)D,
                                              at::cuda::getCurrentCUDAStream().stream(), drop);
  TORCH_CHECK(err == nullptr, "edl attention_varlen_bwd failed: ", err);
}

void check_affine(const Tensor& g, const Tensor& b, int64_t C) {
  TORCH_CHECK(g.is_cuda() && g.scalar_type() == at::kFloat && g.is_contiguous() && g.numel() == C, "gamma: fp32 [C]");
  TORCH_CHECK(b.is_cuda() && b.scalar_type() == at::kFloat && b.is_contiguous() && b.numel() == C, "beta: fp32 [C]");
}

void layernorm_fwd(const Tensor& x, const Tensor& gamma, const Tensor& beta, Tensor& y, double eps) {
  check_bf16_2d(x, "x");
  check_bf16_2d(y, "y");
  const int64_t C = x.size(1);
  TORCH_CHECK(edl::layernorm_supported((int)C) && y.sizes() == x.sizes(), "layernorm: C % 8 == 0, 8 <= C <= 1024");
  check_affine(gamma, beta, C);
  c10::cuda::CUDAGuard guard(x.device());
  edl::layernorm_fwd(x.data_ptr(), gamma.data_ptr<float>(), beta.data_ptr<float>(), y.data_ptr(), x.size(0), (int)C,
                     (float)eps, at::cuda::getCurrentCUDAStream().stream());
}

void embedding_layernorm_fwd(const Tensor& ids, const Tensor& pos_ids, const Tensor& seg_ids, const Tensor& word,
                             const Tensor& pos, const Tensor& seg, const Tensor& gamma, const Tensor& beta, Tensor& y,
                             double eps, Tensor& err, const edl::PhiloxArgs* drop) {
  const int64_t rows = ids.numel();
  for (const Tensor* t : {&ids, &pos_ids, &seg_ids})
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kLong && t->is_contiguous() && t->numel() == rows,
                "ids: contiguous int64 CUDA tensors of one size");
  check_bf16_2d(word, "word");
  check_bf16_2d(pos, "pos");
  check_bf16_2d(seg, "seg");
  check_bf16_2d(y, "y");
  const int64_t C = word.size(1);
  TORCH_CHECK(edl::layernorm_supported((int)C) && pos.size(1) == C && seg.size(1) == C && y.size(0) == rows &&
              y.size(1) == C, "embedding_layernorm: tables and output of one width C, C % 8 == 0, 8 <= C <= 1024");
  check_affine(gamma, beta, C);
  TORCH_CHECK(err.is_cuda() && err.scalar_type() == at::kInt && err.numel() >= 1, "err: int32 CUDA flag");
  c10::cuda::CUDAGuard guard(ids.device());
  edl::embedding_layernorm_fwd(ids.data_ptr<int64_t>(), pos_ids.data_ptr<int64_t>(), seg_ids.data_ptr<int64_t>(),
                               word.data_ptr(), word.size(0), pos.data_ptr(), pos.size(0), seg.data_ptr(), seg.size(0),
                               gamma.data_ptr<float>(), beta.data_ptr<float>(), y.data_ptr(), rows, (int)C, (float)eps,
                               err.data_ptr<int>(), at::cuda::getCurrentCUDAStream().stream(), drop);
}

// x, dy, dx bf16 [rows, C]; part fp32 [layernorm_bwd_ctas(rows) * 2 * C]; dgamma / dbeta fp32 [C]
void layernorm_bwd(const Tensor& x, const Tensor& dy, const Tensor& gamma, Tensor& dx, Tensor& part, Tensor& dgamma,
                   Tensor& dbeta, double eps) {
  for (const Tensor* t : {&x, &dy, static_cast<const Tensor*>(&dx)}) check_bf16_2d(*t, "layernorm_bwd operand");
  const int64_t rows = x.size(0), C = x.size(1);
  TORCH_CHECK(edl::layernorm_supported((int)C) && dy.sizes() == x.sizes() && dx.sizes() == x.sizes(),
              "layernorm_bwd: C % 8 == 0, 8 <= C <= 1024, x / dy / dx of one shape");
  check_affine(dgamma, dbeta, C);
  TORCH_CHECK(gamma.is_cuda() && gamma.scalar_type() == at::kFloat && gamma.is_contiguous() && gamma.numel() == C);
  TORCH_CHECK(part.is_cuda() && part.scalar_type() == at::kFloat && part.is_contiguous() &&
              part.numel() >= (int64_t)edl::layernorm_bwd_ctas(rows) * 2 * C, "part: fp32 [ctas * 2 * C]");
  c10::cuda::CUDAGuard guard(x.device());
  edl::layernorm_bwd(x.data_ptr(), dy.data_ptr(), gamma.data_ptr<float>(), dx.data_ptr(), part.data_ptr<float>(),
                     dgamma.data_ptr<float>(), dbeta.data_ptr<float>(), rows, (int)C, (float)eps,
                     at::cuda::getCurrentCUDAStream().stream());
}

// dE fp32 [rows, C]: the gradient of the gathered row sum of embedding_layernorm_fwd
void embedding_layernorm_bwd(const Tensor& ids, const Tensor& pos_ids, const Tensor& seg_ids, const Tensor& word,
                             const Tensor& pos, const Tensor& seg, const Tensor& dy, const Tensor& gamma, Tensor& dE,
                             Tensor& part, Tensor& dgamma, Tensor& dbeta, double eps, const edl::PhiloxArgs* drop) {
  const int64_t rows = ids.numel();
  for (const Tensor* t : {&ids, &pos_ids, &seg_ids})
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kLong && t->is_contiguous() && t->numel() == rows,
                "ids: contiguous int64 CUDA tensors of one size");
  for (const Tensor* t : {&word, &pos, &seg, &dy}) check_bf16_2d(*t, "embedding_layernorm_bwd operand");
  const int64_t C = word.size(1);
  TORCH_CHECK(edl::layernorm_supported((int)C) && pos.size(1) == C && seg.size(1) == C && dy.size(0) == rows &&
              dy.size(1) == C, "embedding_layernorm_bwd: tables and dy of one width C, C % 8 == 0, 8 <= C <= 1024");
  TORCH_CHECK(dE.is_cuda() && dE.scalar_type() == at::kFloat && dE.is_contiguous() && dE.numel() == rows * C,
              "dE: contiguous fp32 [rows, C]");
  check_affine(dgamma, dbeta, C);
  TORCH_CHECK(gamma.is_cuda() && gamma.scalar_type() == at::kFloat && gamma.is_contiguous() && gamma.numel() == C);
  TORCH_CHECK(part.is_cuda() && part.scalar_type() == at::kFloat && part.is_contiguous() &&
              part.numel() >= (int64_t)edl::layernorm_bwd_ctas(rows) * 2 * C, "part: fp32 [ctas * 2 * C]");
  c10::cuda::CUDAGuard guard(ids.device());
  edl::embedding_layernorm_bwd(ids.data_ptr<int64_t>(), pos_ids.data_ptr<int64_t>(), seg_ids.data_ptr<int64_t>(),
                               word.data_ptr(), word.size(0), pos.data_ptr(), pos.size(0), seg.data_ptr(), seg.size(0),
                               dy.data_ptr(), gamma.data_ptr<float>(), dE.data_ptr<float>(), part.data_ptr<float>(),
                               dgamma.data_ptr<float>(), dbeta.data_ptr<float>(), rows, (int)C, (float)eps,
                               at::cuda::getCurrentCUDAStream().stream(), drop);
}

// q uint8 [rows, C] (contiguous), sa fp32 [ceil(C/128), rows]: the block quantisation of the stored y
void check_quant_out(const Tensor& y, const Tensor& q, const Tensor& sa) {
  const int64_t rows = y.size(0), C = y.size(1);
  TORCH_CHECK(q.is_cuda() && q.device() == y.device() && q.element_size() == 1 && q.is_contiguous() && q.dim() == 2 &&
              q.size(0) == rows && q.size(1) == C && reinterpret_cast<uintptr_t>(q.data_ptr()) % 8 == 0,
              "q must be a contiguous, 8-byte aligned 1-byte [rows, C] tensor");
  TORCH_CHECK(sa.is_cuda() && sa.device() == y.device() && sa.scalar_type() == at::kFloat && sa.is_contiguous() &&
              sa.dim() == 2 && sa.size(0) == (C + 127) / 128 && sa.size(1) == rows,
              "sa must be contiguous fp32 [ceil(C/128), rows]");
}

void layernorm_e4m3_fwd(const Tensor& x, const Tensor& gamma, const Tensor& beta, Tensor& y, Tensor& q, Tensor& sa,
                        double eps) {
  check_bf16_2d(x, "x");
  check_bf16_2d(y, "y");
  const int64_t C = x.size(1);
  TORCH_CHECK(edl::layernorm_supported((int)C) && y.sizes() == x.sizes(), "layernorm: C % 8 == 0, 8 <= C <= 1024");
  check_affine(gamma, beta, C);
  check_quant_out(y, q, sa);
  c10::cuda::CUDAGuard guard(x.device());
  edl::layernorm_e4m3_fwd(x.data_ptr(), gamma.data_ptr<float>(), beta.data_ptr<float>(), y.data_ptr(), q.data_ptr(),
                          sa.data_ptr<float>(), x.size(0), (int)C, (float)eps, at::cuda::getCurrentCUDAStream().stream());
}

void embedding_layernorm_e4m3_fwd(const Tensor& ids, const Tensor& pos_ids, const Tensor& seg_ids, const Tensor& word,
                                  const Tensor& pos, const Tensor& seg, const Tensor& gamma, const Tensor& beta,
                                  Tensor& y, Tensor& q, Tensor& sa, double eps, Tensor& err) {
  const int64_t rows = ids.numel();
  for (const Tensor* t : {&ids, &pos_ids, &seg_ids})
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kLong && t->is_contiguous() && t->numel() == rows,
                "ids: contiguous int64 CUDA tensors of one size");
  check_bf16_2d(word, "word");
  check_bf16_2d(pos, "pos");
  check_bf16_2d(seg, "seg");
  check_bf16_2d(y, "y");
  const int64_t C = word.size(1);
  TORCH_CHECK(edl::layernorm_supported((int)C) && pos.size(1) == C && seg.size(1) == C && y.size(0) == rows &&
              y.size(1) == C, "embedding_layernorm: tables and output of one width C, C % 8 == 0, 8 <= C <= 1024");
  check_affine(gamma, beta, C);
  check_quant_out(y, q, sa);
  TORCH_CHECK(err.is_cuda() && err.scalar_type() == at::kInt && err.numel() >= 1, "err: int32 CUDA flag");
  c10::cuda::CUDAGuard guard(ids.device());
  edl::embedding_layernorm_e4m3_fwd(ids.data_ptr<int64_t>(), pos_ids.data_ptr<int64_t>(), seg_ids.data_ptr<int64_t>(),
                                    word.data_ptr(), word.size(0), pos.data_ptr(), pos.size(0), seg.data_ptr(),
                                    seg.size(0), gamma.data_ptr<float>(), beta.data_ptr<float>(), y.data_ptr(),
                                    q.data_ptr(), sa.data_ptr<float>(), rows, (int)C, (float)eps, err.data_ptr<int>(),
                                    at::cuda::getCurrentCUDAStream().stream());
}

}  // namespace

void register_transformer_bindings(pybind11::module_& m) {
  // a drawn dropout site; seed / offset are the values the kernels use (0 when captured: then read at run time)
  pybind11::class_<edl::PhiloxArgs>(m, "PhiloxArgs")
      .def_readonly("seed", &edl::PhiloxArgs::seed)
      .def_readonly("offset", &edl::PhiloxArgs::offset)
      .def_readonly("threshold", &edl::PhiloxArgs::threshold)
      .def_readonly("scale", &edl::PhiloxArgs::scale)
      .def_property_readonly("captured", [](const edl::PhiloxArgs& a) { return a.seed_ptr != nullptr; });
  m.def("dropout_draw", &dropout_draw);
  m.def("dropout_fwd", &dropout_fwd);
  m.def("attention_fwd", &attention_fwd);
  m.def("attention_supported", &edl::attention_supported);
  m.def("attention_varlen_fwd", &attention_varlen_fwd);
  m.def("attention_varlen_supported", &edl::attention_varlen_supported);
  m.def("attention_varlen_bwd", &attention_varlen_bwd);
  m.def("layernorm_fwd", &layernorm_fwd);
  m.def("layernorm_supported", &edl::layernorm_supported);
  m.def("attention_bwd", &attention_bwd);
  m.def("layernorm_bwd", &layernorm_bwd);
  m.def("layernorm_bwd_ctas", &edl::layernorm_bwd_ctas);
  m.def("embedding_layernorm_bwd", &embedding_layernorm_bwd);
  m.def("embedding_layernorm_fwd", &embedding_layernorm_fwd);
  m.def("layernorm_e4m3_fwd", &layernorm_e4m3_fwd);
  m.def("embedding_layernorm_e4m3_fwd", &embedding_layernorm_e4m3_fwd);
}
