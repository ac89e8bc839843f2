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

// t, or a copy of it when it does not start on 16 bytes (TMA boxes and the kernels' vector loads need that start)
Tensor aligned16(const Tensor& t) { return reinterpret_cast<uintptr_t>(t.data_ptr()) % 16 == 0 ? t : t.clone(); }

const uint16_t* opt_bias(const c10::optional<Tensor>& bias, int64_t n, Tensor& keep) {
  if (bias.has_value() && bias->defined()) {
    keep = bias->to(at::kBFloat16).contiguous();
    TORCH_CHECK(keep.numel() == n, "ao_b200: bias must have N elements");
    return bf16_ptr(keep);
  }
  return nullptr;
}

// bf16 activations may be row-strided (a column slice of a wider buffer); returns the row pitch in elements
int64_t check_rows(const Tensor& x, const char* name) {
  TORCH_CHECK(x.is_cuda(), "ao_b200: ", name, " must be a CUDA tensor");
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && x.dim() == 2, "ao_b200: ", name, " must be bf16 [M, K]");
  TORCH_CHECK(x.size(1) <= 1 || x.stride(1) == 1, "ao_b200: ", name, " must have unit inner stride");
  TORCH_CHECK(x.size(0) <= 1 || (x.stride(0) >= x.size(1) && x.stride(0) % 8 == 0), "ao_b200: the row pitch of ", name,
              " must be >= K and a multiple of 8 elements");
  TORCH_CHECK(reinterpret_cast<uintptr_t>(x.data_ptr()) % 16 == 0, "ao_b200: ", name, " must be 16-byte aligned");
  return x.size(0) > 1 ? x.stride(0) : x.size(1);
}

// A dense linear as every such op runs it once it has checked its own operands and allocated y [M, n_out] through its
// Meta kernel.  The activation x [M, K] has passed one of two rules: bf16 rows check_rows (strided rows keep their
// pitch, a start off 16 bytes is rejected); quantized codes check_cuda (contiguous), and codes that do not start on 16
// bytes are copied here.  launch(x, ldx, bias, y, ws, ws_bytes) makes the op's C call; without rows there is none.
template <class Launch>
Tensor dense_linear(const Tensor& x, const c10::optional<Tensor>& bias, Tensor y, Launch launch) {
  c10::cuda::CUDAGuard guard(x.device());
  Tensor keep;
  const uint16_t* b = opt_bias(bias, y.size(1), keep);
  if (x.size(0) == 0) return y;
  const Tensor xc = aligned16(x);
  const int64_t ldx = xc.size(0) > 1 ? xc.stride(0) : xc.size(1);
  Tensor ws = workspace_for(x);
  launch(xc.data_ptr(), (int)ldx, b, y.data_ptr(), ws.data_ptr(), (size_t)ws.numel());
  return y;
}

// torch._grouped_mm(x, W.transpose(-2, -1), offs), 2-D x 3-D, as every grouped op runs it once it has checked its own
// operands: x [M, K] on the GPU, w the experts' weights [E, ...], offs int32 [E] on x's device (cumulative row ends,
// never read on the host) -> y [M, n_out] bf16.  The kernels read dense rows from a 16-byte aligned start, so an x
// that is not (a column slice, a view at an odd storage offset) is copied.  launch(x, y, ws, ws_bytes) makes the op's
// C call; without rows there is none.
template <class Launch>
Tensor grouped_mm(const Tensor& x, const char* name, const Tensor& w, const Tensor& offs, int64_t n_out, Launch launch) {
  TORCH_CHECK(x.is_cuda(), "ao_b200: ", name, " must be a CUDA tensor");
  check_cuda(offs, "offs");
  TORCH_CHECK(offs.scalar_type() == at::kInt && offs.dim() == 1 && offs.size(0) == w.size(0),
              "ao_b200: offs must be int32 [E], E=", w.size(0));
  TORCH_CHECK(offs.device() == x.device(), "ao_b200: offs must be on the device of ", name);
  c10::cuda::CUDAGuard guard(x.device());
  Tensor y = at::empty({x.size(0), n_out}, x.options().dtype(at::kBFloat16));
  if (x.size(0) == 0) return y;
  const Tensor xc = aligned16(x.contiguous());
  Tensor ws = workspace_for(x);
  launch(xc.data_ptr(), bf16_ptr_mut(y), ws.data_ptr(), (size_t)ws.numel());
  return y;
}

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
Tensor int4_tilepacked_linear_meta(const Tensor& x, const Tensor& qdata, int64_t, const Tensor&,
                                   const c10::optional<Tensor>&, int64_t n_out, int64_t) {
  if (n_out <= 0) n_out = qdata.size(0) * 8;
  return at::empty({x.size(0), n_out}, x.options());
}
Tensor int4_tilepacked_linear(const Tensor& x, const Tensor& qdata, int64_t group_size,
                              const Tensor& scale_and_zero, const c10::optional<Tensor>& bias,
                              int64_t n_out, int64_t impl) {
  check_rows(x, "x");
  check_cuda(qdata, "qdata");
  check_cuda(scale_and_zero, "scale_and_zero");
  TORCH_CHECK(qdata.scalar_type() == at::kInt && qdata.dim() == 4 && qdata.size(2) == 32 && qdata.size(3) == 4, "ao_b200: qdata must be int32 [N/8, K/128, 32, 4] (inner_k_tiles=8)");
  TORCH_CHECK(scale_and_zero.scalar_type() == at::kBFloat16 && scale_and_zero.dim() == 3 && scale_and_zero.size(2) == 2, "ao_b200: scale_and_zero must be bf16 [K/g, N, 2]");
  const int64_t M = x.size(0), K = x.size(1);
  const int64_t N = qdata.size(0) * 8;
  TORCH_CHECK(qdata.size(1) * 128 == K, "ao_b200: x has K=", K, " but qdata encodes K=", qdata.size(1) * 128);
  TORCH_CHECK(scale_and_zero.size(0) * group_size == K && scale_and_zero.size(1) == N, "ao_b200: scale_and_zero shape does not match (K/g, N)");
  TORCH_CHECK(n_out <= N, "ao_b200: n_out > N");
  Tensor y = int4_tilepacked_linear_meta(x, qdata, group_size, scale_and_zero, bias, n_out, impl);
  return dense_linear(x, bias, y, [&](const void* xp, int ldx, const uint16_t* b, void* yp, void* ws, size_t ws_bytes) {
    AO_CALL(ao_int4_tilepacked_linear_strided(static_cast<const uint16_t*>(xp), ldx, (int)M, (int)K, qdata.data_ptr<int32_t>(), bf16_ptr(scale_and_zero), (int)group_size, (int)N, b, static_cast<uint16_t*>(yp), (int)y.size(1), ws, ws_bytes, (int)impl, cur_stream()));
  });
}

// torch._grouped_mm on 3-D int4 expert weights (2-D x 3-D): x bf16 [M, K], qdata int32 [E, N/8, K/128, 32, 4],
// scale_and_zero bf16 [E, K/g, N, 2], offs int32 [E] -> y [M, n_out] (n_out <= 0: N).  Rows from offs[E-1] on are left
// unwritten, as torch leaves them.
Tensor int4_tilepacked_grouped_mm(const Tensor& x, const Tensor& qdata, int64_t group_size, const Tensor& scale_and_zero,
                                  const Tensor& offs, int64_t n_out) {
  check_cuda(qdata, "qdata");
  check_cuda(scale_and_zero, "scale_and_zero");
  TORCH_CHECK(x.scalar_type() == at::kBFloat16 && x.dim() == 2, "ao_b200: x must be bf16 [M, K]");
  TORCH_CHECK(qdata.scalar_type() == at::kInt && qdata.dim() == 5 && qdata.size(3) == 32 && qdata.size(4) == 4, "ao_b200: qdata must be int32 [E, N/8, K/128, 32, 4]");
  TORCH_CHECK(scale_and_zero.scalar_type() == at::kBFloat16 && scale_and_zero.dim() == 4 && scale_and_zero.size(3) == 2, "ao_b200: scale_and_zero must be bf16 [E, K/g, N, 2]");
  const int64_t M = x.size(0), K = x.size(1), E = qdata.size(0), N = qdata.size(1) * 8;
  TORCH_CHECK(qdata.size(2) * 128 == K, "ao_b200: x has K=", K, " but qdata encodes K=", qdata.size(2) * 128);
  TORCH_CHECK(scale_and_zero.size(0) == E && scale_and_zero.size(1) * group_size == K && scale_and_zero.size(2) == N, "ao_b200: scale_and_zero shape does not match (E, K/g, N)");
  if (n_out <= 0) n_out = N;
  TORCH_CHECK(n_out <= N, "ao_b200: n_out > N");
  return grouped_mm(x, "x", qdata, offs, n_out, [&](const void* xc, uint16_t* y, void* ws, size_t ws_bytes) {
    AO_CALL(ao_int4_tilepacked_grouped_mm(static_cast<const uint16_t*>(xc), (int)M, (int)K, qdata.data_ptr<int32_t>(), bf16_ptr(scale_and_zero), (int)group_size, (int)E, (int)N, (int)n_out, offs.data_ptr<int32_t>(), y, ws, ws_bytes, cur_stream()));
  });
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
Tensor int4_tilepacked_grouped_mm_meta(const Tensor& x, const Tensor& qdata, int64_t, const Tensor&, const Tensor&,
                                       int64_t n_out) {
  if (n_out <= 0) n_out = qdata.size(1) * 8;
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
  m.def("int4_tilepacked_grouped_mm(Tensor x, Tensor qdata, int group_size, Tensor scale_and_zero, Tensor offs, int n_out) -> Tensor");
  m.def("launch_count() -> int", []() -> int64_t { return (int64_t)ao_b200_launch_count(); });
  m.def("debug_workspace(Tensor like) -> Tensor", [](const at::Tensor& like) { return workspace_for(like); });
  // tests only: force the stream-K grid of every GEMM launch (0 = heuristic); returns the previous value
  m.def("debug_set_streamk_ctas(int n) -> int", [](int64_t n) -> int64_t { return ao_b200_debug_set_streamk_ctas((int)n); });
  // on the current device's current stream: orders a weight written by the quantizers before the linears that read it
  m.def("pdl_fence() -> ()", []() { AO_CALL(ao_b200_pdl_fence(cur_stream())); });
  ao_b200_define_lowp(m);
}

TORCH_LIBRARY_IMPL(ao_b200, CUDA, m) {
  m.impl("int4_pack_tile4d", &int4_pack_tile4d);
  m.impl("int4_unpack_tile4d", &int4_unpack_tile4d);
  m.impl("int4_dequant_tile4d", &int4_dequant_tile4d);
  m.impl("int4_hqq_quantize", &int4_hqq_quantize);
  m.impl("int4_tilepacked_linear", &int4_tilepacked_linear);
  m.impl("int4_tilepacked_grouped_mm", &int4_tilepacked_grouped_mm);
  ao_b200_impl_lowp_cuda(m);
}

TORCH_LIBRARY_IMPL(ao_b200, Meta, m) {
  m.impl("int4_pack_tile4d", &int4_pack_tile4d_meta);
  m.impl("int4_unpack_tile4d", &int4_unpack_tile4d_meta);
  m.impl("int4_dequant_tile4d", &int4_dequant_tile4d_meta);
  m.impl("int4_hqq_quantize", &int4_hqq_quantize_meta);
  m.impl("int4_tilepacked_linear", &int4_tilepacked_linear_meta);
  m.impl("int4_tilepacked_grouped_mm", &int4_tilepacked_grouped_mm_meta);
  ao_b200_impl_lowp_meta(m);
}
