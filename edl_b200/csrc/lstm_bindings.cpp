// torch bindings for the bidirectional LSTM recurrence (lstm.cu).
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/extension.h>

#include "kernels.h"

namespace {
using torch::Tensor;

void check(const Tensor& t, at::ScalarType st, std::initializer_list<int64_t> shape, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == st && t.is_contiguous() && t.sizes().equals(shape) &&
                  reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0,
              name, ": contiguous, 16-byte aligned CUDA tensor of the expected dtype and shape");
}

constexpr int64_t H = edl::kLstmHidden;

void lstm_fwd(const Tensor& xproj, const Tensor& whh, const Tensor& lengths, Tensor& hs, Tensor& hn, Tensor& gates,
              Tensor& cs, int64_t L) {
  const int64_t B = lengths.numel();
  TORCH_CHECK(edl::lstm_supported((int)B, (int)L, 8, (int)H), "lstm_fwd: unsupported shape");
  check(lengths, at::kInt, {B}, "lengths");
  check(xproj, at::kBFloat16, {L * B, 8 * H}, "xproj");
  check(whh, at::kBFloat16, {2, 4 * H, H}, "whh");
  check(hs, at::kBFloat16, {(L + 2) * B, 2 * H}, "hs");
  check(hn, at::kBFloat16, {2, B, H}, "hn");
  check(gates, at::kBFloat16, {L * B, 2, H, 4}, "gates");
  check(cs, at::kFloat, {L * B, 2, H}, "cs");
  c10::cuda::CUDAGuard guard(xproj.device());
  const char* err = edl::lstm_fwd(xproj.data_ptr(), whh.data_ptr(), lengths.data_ptr<int>(), hs.data_ptr(),
                                  hn.data_ptr(), gates.data_ptr(), cs.data_ptr<float>(), (int)B, (int)L,
                                  at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl lstm_fwd failed: ", err);
}

// dy: bf16 [B, L, 2H] with unit stride in the last dimension and even strides, or None; dhn: bf16 [2, B, H] or None
void lstm_bwd(const Tensor& whh, const Tensor& lengths, const Tensor& gates, const Tensor& cs,
              const c10::optional<Tensor>& dy, const c10::optional<Tensor>& dhn, Tensor& dgates, int64_t L) {
  const int64_t B = lengths.numel();
  TORCH_CHECK(edl::lstm_supported((int)B, (int)L, 8, (int)H), "lstm_bwd: unsupported shape");
  check(lengths, at::kInt, {B}, "lengths");
  check(whh, at::kBFloat16, {2, 4 * H, H}, "whh");
  check(gates, at::kBFloat16, {L * B, 2, H, 4}, "gates");
  check(cs, at::kFloat, {L * B, 2, H}, "cs");
  check(dgates, at::kBFloat16, {L * B, 8 * H}, "dgates");
  const void* dyp = nullptr;
  int64_t sb = 0, st = 0;
  if (dy.has_value() && dy->defined()) {
    TORCH_CHECK(dy->is_cuda() && dy->scalar_type() == at::kBFloat16 && dy->dim() == 3 && dy->size(0) == B &&
                    dy->size(1) == L && dy->size(2) == 2 * H && dy->stride(2) == 1 && dy->stride(0) % 2 == 0 &&
                    dy->stride(1) % 2 == 0 && reinterpret_cast<uintptr_t>(dy->data_ptr()) % 4 == 0,
                "dy: bf16 [B, L, 2H], unit stride in the last dimension, even strides, 4-byte aligned");
    dyp = dy->data_ptr();
    sb = dy->stride(0);
    st = dy->stride(1);
  }
  const void* dhp = nullptr;
  if (dhn.has_value() && dhn->defined()) {
    check(*dhn, at::kBFloat16, {2, B, H}, "dhn");
    dhp = dhn->data_ptr();
  }
  c10::cuda::CUDAGuard guard(whh.device());
  const char* err = edl::lstm_bwd(whh.data_ptr(), lengths.data_ptr<int>(), gates.data_ptr(), cs.data_ptr<float>(), dyp,
                                  sb, st, dhp, dgates.data_ptr(), (int)B, (int)L,
                                  at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(err == nullptr, "edl lstm_bwd failed: ", err);
}

}  // namespace

void register_lstm_bindings(pybind11::module_& m) {
  m.def("lstm_fwd", &lstm_fwd);
  m.def("lstm_bwd", &lstm_bwd);
  m.def("lstm_supported", &edl::lstm_supported);
}
