// torch.library registration of the C-ABI kernels as torch.ops.ao_b200.* (CUDA + Meta).
// This is the layer the reference fills with torch.library.Library("torchao", "FRAGMENT")
// defs + TORCH_LIBRARY_IMPL(torchao, CUDA, ...) (torchao/ops.py:12-49,
// torchao/csrc/cuda/mx_kernels/mxfp8_extension.cpp:425-429).  Ops are functional
// (allocate and return their outputs), validate with TORCH_CHECK, launch on the current
// CUDA stream under a device guard, never synchronise and are CUDA-graph capturable.
#include <ATen/ATen.h>
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <torch/library.h>

#include <map>
#include <mutex>
#include <tuple>

#include "ao_b200.h"

namespace {

using at::Tensor;

#define AO_CALL(expr)                                                                   \
  do {                                                                                  \
    int _rc = (expr);                                                                   \
    TORCH_CHECK(_rc == AO_OK, "ao_b200: ", #expr, " failed (", _rc, "): ", ao_b200_last_error()); \
  } while (0)

void* cur_stream() { return (void*)at::cuda::getCurrentCUDAStream().stream(); }

// split-K scratch: one zero-initialised buffer per (device, stream).
Tensor workspace_for(const Tensor& like) {
  static std::mutex mu;
  static std::map<std::pair<int, void*>, Tensor> cache;
  const int dev = like.get_device();
  void* st = cur_stream();
  std::lock_guard<std::mutex> lock(mu);
  auto it = cache.find({dev, st});
  if (it != cache.end()) return it->second;
  const int64_t bytes = (int64_t)ao_b200_workspace_bytes(0, 0);
  Tensor ws = at::zeros({bytes}, like.options().dtype(at::kByte));
  cache[{dev, st}] = ws;
  return ws;
}

void check_cuda(const Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda(), "ao_b200: ", name, " must be a CUDA tensor");
  TORCH_CHECK(t.is_contiguous(), "ao_b200: ", name, " must be contiguous");
}

const uint16_t* bf16_ptr(const Tensor& t) { return reinterpret_cast<const uint16_t*>(t.data_ptr()); }
uint16_t* bf16_ptr_mut(Tensor& t) { return reinterpret_cast<uint16_t*>(t.data_ptr()); }

// ------------------------------------------------------------------ int4
Tensor int4_pack_tile4d(const Tensor& q_u8, int64_t inner_k_tiles) {
  check_cuda(q_u8, "q_u8");
  TORCH_CHECK(q_u8.scalar_type() == at::kByte && q_u8.dim() == 2, "ao_b200: q_u8 must be uint8 [N, K/2]");
  c10::cuda::CUDAGuard guard(q_u8.device());
  const int64_t N = q_u8.size(0), K = q_u8.size(1) * 2;
  TORCH_CHECK(N % 8 == 0 && K % (inner_k_tiles * 16) == 0, "ao_b200: int4 pack needs N%8==0 and K%(inner_k_tiles*16)==0, got N=", N, " K=", K);
  Tensor out = at::empty({N / 8, K / (inner_k_tiles * 16), 32, inner_k_tiles / 2}, q_u8.options().dtype(at::kInt));
  AO_CALL(ao_int4_pack_tile4d(q_u8.data_ptr<uint8_t>(), out.data_ptr<int32_t>(), (int)N, (int)K, (int)inner_k_tiles, cur_stream()));
  return out;
}

Tensor int4_unpack_tile4d(const Tensor& qdata) {
  check_cuda(qdata, "qdata");
  TORCH_CHECK(qdata.scalar_type() == at::kInt && qdata.dim() == 4 && qdata.size(2) == 32, "ao_b200: qdata must be int32 [N/8, K/(ikt*16), 32, ikt/2]");
  c10::cuda::CUDAGuard guard(qdata.device());
  const int64_t ikt = qdata.size(3) * 2;
  const int64_t N = qdata.size(0) * 8, K = qdata.size(1) * ikt * 16;
  Tensor out = at::empty({N, K / 2}, qdata.options().dtype(at::kByte));
  AO_CALL(ao_int4_unpack_tile4d(qdata.data_ptr<int32_t>(), out.data_ptr<uint8_t>(), (int)N, (int)K, (int)ikt, cur_stream()));
  return out;
}

Tensor int4_dequant_tile4d(const Tensor& qdata, const Tensor& scale_and_zero, int64_t group_size) {
  check_cuda(qdata, "qdata");
  check_cuda(scale_and_zero, "scale_and_zero");
  TORCH_CHECK(qdata.scalar_type() == at::kInt && qdata.dim() == 4 && qdata.size(2) == 32 && qdata.size(3) == 4, "ao_b200: qdata must be int32 [N/8, K/128, 32, 4]");
  TORCH_CHECK(scale_and_zero.scalar_type() == at::kBFloat16 && scale_and_zero.dim() == 3, "ao_b200: scale_and_zero must be bf16 [K/g, N, 2]");
  c10::cuda::CUDAGuard guard(qdata.device());
  const int64_t N = qdata.size(0) * 8, K = qdata.size(1) * 128;
  TORCH_CHECK(scale_and_zero.size(0) == K / group_size && scale_and_zero.size(1) == N, "ao_b200: scale_and_zero shape mismatch");
  Tensor out = at::empty({N, K}, scale_and_zero.options());
  AO_CALL(ao_int4_dequant_tile4d(qdata.data_ptr<int32_t>(), bf16_ptr(scale_and_zero), bf16_ptr_mut(out), (int)N, (int)K, (int)group_size, cur_stream()));
  return out;
}

// w bf16 [N, K] -> (q uint8 [N, K], scale bf16 [N, K/g], zero bf16 [N, K/g])  (HQQ solver, tinygemm convention)
std::tuple<Tensor, Tensor, Tensor> int4_hqq_quantize(const Tensor& w, int64_t group_size) {
  check_cuda(w, "w");
  TORCH_CHECK(w.scalar_type() == at::kBFloat16 && w.dim() == 2, "ao_b200: w must be bf16 [N, K]");
  c10::cuda::CUDAGuard guard(w.device());
  const int64_t N = w.size(0), K = w.size(1);
  TORCH_CHECK(K % group_size == 0, "ao_b200: K=", K, " must be a multiple of group_size=", group_size);
  Tensor q = at::empty({N, K}, w.options().dtype(at::kByte));
  Tensor s = at::empty({N, K / group_size}, w.options());
  Tensor z = at::empty({N, K / group_size}, w.options());
  Tensor ws = at::empty({(int64_t)ao_int4_hqq_workspace_bytes((int)N, (int)K, (int)group_size)}, w.options().dtype(at::kByte));
  AO_CALL(ao_int4_hqq_quantize(bf16_ptr(w), (int)N, (int)K, (int)group_size, q.data_ptr<uint8_t>(), bf16_ptr_mut(s),
                               bf16_ptr_mut(z), ws.data_ptr(), (size_t)ws.numel(), cur_stream()));
  return {q, s, z};
}
std::tuple<Tensor, Tensor, Tensor> int4_hqq_quantize_meta(const Tensor& w, int64_t group_size) {
  return {at::empty({w.size(0), w.size(1)}, w.options().dtype(at::kByte)),
          at::empty({w.size(0), w.size(1) / group_size}, w.options()), at::empty({w.size(0), w.size(1) / group_size}, w.options())};
}

// x [M, K] bf16 -> y [M, n_out] bf16  (aten._weight_int4pack_mm + bias + out-feature slice)
Tensor int4_tilepacked_linear(const Tensor& x, const Tensor& qdata, int64_t group_size,
                              const Tensor& scale_and_zero, const c10::optional<Tensor>& bias,
                              int64_t n_out, int64_t impl) {
  TORCH_CHECK(x.is_cuda(), "ao_b200: x must be a CUDA tensor");
  check_cuda(qdata, "qdata");
  check_cuda(scale_and_zero, "scale_and_zero");
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && x.dim() == 2, "ao_b200: x must be bf16 [M, K]");
  // rows may be strided (a column slice of a wider buffer): the TMA descriptor carries the pitch
  TORCH_CHECK(x.size(1) <= 1 || x.stride(1) == 1, "ao_b200: x must have unit inner stride");
  TORCH_CHECK(x.size(0) <= 1 || (x.stride(0) >= x.size(1) && x.stride(0) % 8 == 0),
              "ao_b200: the row pitch of x must be >= K and a multiple of 8 elements");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0, "ao_b200: x must be 16-byte aligned");
  TORCH_CHECK(qdata.scalar_type() == at::kInt && qdata.dim() == 4 && qdata.size(2) == 32 && qdata.size(3) == 4, "ao_b200: qdata must be int32 [N/8, K/128, 32, 4] (inner_k_tiles=8)");
  TORCH_CHECK(scale_and_zero.scalar_type() == at::kBFloat16 && scale_and_zero.dim() == 3 && scale_and_zero.size(2) == 2, "ao_b200: scale_and_zero must be bf16 [K/g, N, 2]");
  c10::cuda::CUDAGuard guard(x.device());
  const int64_t M = x.size(0), K = x.size(1);
  const int64_t N = qdata.size(0) * 8;
  TORCH_CHECK(qdata.size(1) * 128 == K, "ao_b200: x has K=", K, " but qdata encodes K=", qdata.size(1) * 128);
  TORCH_CHECK(scale_and_zero.size(0) * group_size == K && scale_and_zero.size(1) == N, "ao_b200: scale_and_zero shape does not match (K/g, N)");
  if (n_out <= 0) n_out = N;
  TORCH_CHECK(n_out <= N, "ao_b200: n_out > N");
  const uint16_t* bias_p = nullptr;
  Tensor bias_c;
  if (bias.has_value() && bias->defined()) {
    bias_c = bias->to(at::kBFloat16).contiguous();
    TORCH_CHECK(bias_c.numel() == n_out, "ao_b200: bias must have n_out elements");
    bias_p = bf16_ptr(bias_c);
  }
  Tensor y = at::empty({M, n_out}, x.options());
  if (M == 0) return y;
  Tensor ws = workspace_for(x);
  const int64_t ldx = M > 1 ? x.stride(0) : K;
  AO_CALL(ao_int4_tilepacked_linear_strided(bf16_ptr(x), (int)ldx, (int)M, (int)K, qdata.data_ptr<int32_t>(), bf16_ptr(scale_and_zero), (int)group_size, (int)N, bias_p, bf16_ptr_mut(y), (int)n_out, ws.data_ptr(), (size_t)ws.numel(), (int)impl, cur_stream()));
  return y;
}

// ------------------------------------------------------------------ meta kernels
Tensor int4_pack_tile4d_meta(const Tensor& q_u8, int64_t ikt) {
  return at::empty({q_u8.size(0) / 8, q_u8.size(1) * 2 / (ikt * 16), 32, ikt / 2}, q_u8.options().dtype(at::kInt));
}
Tensor int4_unpack_tile4d_meta(const Tensor& qdata) {
  const int64_t ikt = qdata.size(3) * 2;
  return at::empty({qdata.size(0) * 8, qdata.size(1) * ikt * 8}, qdata.options().dtype(at::kByte));
}
Tensor int4_dequant_tile4d_meta(const Tensor& qdata, const Tensor& sz, int64_t) {
  return at::empty({qdata.size(0) * 8, qdata.size(1) * 128}, sz.options());
}
Tensor int4_tilepacked_linear_meta(const Tensor& x, const Tensor& qdata, int64_t, const Tensor&,
                                   const c10::optional<Tensor>&, int64_t n_out, int64_t) {
  if (n_out <= 0) n_out = qdata.size(0) * 8;
  return at::empty({x.size(0), n_out}, x.options());
}

}  // namespace

#include "torch_binding_lowp.inc"

TORCH_LIBRARY(ao_b200, m) {
  m.def("int4_pack_tile4d(Tensor q_u8, int inner_k_tiles) -> Tensor");
  m.def("int4_unpack_tile4d(Tensor qdata) -> Tensor");
  m.def("int4_dequant_tile4d(Tensor qdata, Tensor scale_and_zero, int group_size) -> Tensor");
  m.def("int4_hqq_quantize(Tensor w, int group_size) -> (Tensor, Tensor, Tensor)");
  m.def("int4_tilepacked_linear(Tensor x, Tensor qdata, int group_size, Tensor scale_and_zero, Tensor? bias, int n_out=0, int impl=0) -> Tensor");
  m.def("launch_count() -> int", []() -> int64_t { return (int64_t)ao_b200_launch_count(); });
  m.def("debug_workspace(Tensor like) -> Tensor", [](const at::Tensor& like) { return workspace_for(like); });
  // tests only: force the stream-K grid of every GEMM launch (0 = heuristic); returns the previous value
  m.def("debug_set_streamk_ctas(int n) -> int", [](int64_t n) -> int64_t { return ao_b200_debug_set_streamk_ctas((int)n); });
  ao_b200_define_lowp(m);
}

TORCH_LIBRARY_IMPL(ao_b200, CUDA, m) {
  m.impl("int4_pack_tile4d", &int4_pack_tile4d);
  m.impl("int4_unpack_tile4d", &int4_unpack_tile4d);
  m.impl("int4_dequant_tile4d", &int4_dequant_tile4d);
  m.impl("int4_hqq_quantize", &int4_hqq_quantize);
  m.impl("int4_tilepacked_linear", &int4_tilepacked_linear);
  ao_b200_impl_lowp_cuda(m);
}

TORCH_LIBRARY_IMPL(ao_b200, Meta, m) {
  m.impl("int4_pack_tile4d", &int4_pack_tile4d_meta);
  m.impl("int4_unpack_tile4d", &int4_unpack_tile4d_meta);
  m.impl("int4_dequant_tile4d", &int4_dequant_tile4d_meta);
  m.impl("int4_hqq_quantize", &int4_hqq_quantize_meta);
  m.impl("int4_tilepacked_linear", &int4_tilepacked_linear_meta);
  ao_b200_impl_lowp_meta(m);
}
