/*
 * ao_b200.h — C ABI of the H100-native quantized-linear engine (libao_b200.so).
 *
 * This is the drop-in boundary for the quantized nn.Linear forward of pytorch/ao
 * (torchao 0.19).  Every entry point replaces one kernel-level call the reference
 * makes from its tensor-subclass linear handlers; the reference file:line each one
 * stands in for is cited beside it.  Signatures are plain device pointers, sizes
 * and a CUDA stream: no torch types.  The torch.library registration that binds
 * these as torch.ops.ao_b200.* lives in ao_b200/csrc/torch_binding.cpp.
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless the name ends in _host;
 *   - `stream` is a cudaStream_t passed as void* (NULL = legacy default stream);
 *   - matrices are row-major; a linear is Y[M,N] = X[M,K] * W[N,K]^T (+ bias[N]);
 *   - bf16 values are passed as uint16_t bit patterns;
 *   - return value: 0 on success, negative AO_ERR_* otherwise, with a message
 *     retrievable from ao_b200_last_error() (thread-local);
 *   - kernels never synchronise the device and are CUDA-graph capturable
 *     (tensor maps are built on the host and passed by value);
 *   - `workspace` is caller-owned scratch for split-K partials + flags; it
 *     must be zero-initialised once (kernels restore the flags to zero) and
 *     must not be shared by linears running concurrently on different streams;
 *   - kernels are launched with programmatic dependent launch (PDL): each one
 *     lets the next kernel on the stream start early and waits for its
 *     predecessor before reading activations, scales, offs or the workspace.
 *     The dense GEMMs behind every linear below request their first WEIGHT
 *     tiles (wq and the weight scales) before that wait, so weights must be
 *     complete before the GEMM's predecessor starts.  A buffer written by this
 *     library's quantizers (ao_*_quantize*) and then read as the weights of a
 *     linear must be separated from that linear by ao_b200_pdl_fence, by any
 *     launch without PDL (e.g. a torch kernel) or by an event / stream sync.
 *     The grouped GEMMs read no weight before the wait.
 */
#ifndef AO_B200_H_
#define AO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AO_OK 0
#define AO_ERR_INVALID_ARG (-1)
#define AO_ERR_CUDA (-2)
#define AO_ERR_UNSUPPORTED (-3)
#define AO_ERR_WORKSPACE (-4)

/* library / device ---------------------------------------------------------- */
int ao_b200_version(void);
const char* ao_b200_last_error(void);
/* 1 when the current device is compute capability 9.0 (sm_90a kernels can run). */
int ao_b200_device_ok(void);
/* bytes of workspace any linear below may need for (M, N) outputs. */
size_t ao_b200_workspace_bytes(int M, int N);
/* number of kernels this library has launched since load (bench.py "gpu_launches"). */
uint64_t ao_b200_launch_count(void);
/* TEST ONLY: force the CTA count of the stream-K GEMM kernel behind every linear below, so that tests can reach
 * every split-tile pattern on any SM count.  n > 0 launches clamp(n, 1, min(SM count, work units)) CTAs, n = 0
 * restores the per-problem heuristic.  Process-wide, not thread-safe against concurrent launches; returns the
 * previous value.  No production path calls it. */
int ao_b200_debug_set_streamk_ctas(int n);
/* Launches one empty kernel without PDL that never lets its dependents start early: the next kernel on `stream` starts
 * only after every kernel before the fence has completed and its writes are visible.  Call it between quantizing a
 * weight with this library and the first linear that reads it (quantize_ does). */
int ao_b200_pdl_fence(void* stream);

/* int4 weight-only, tile_packed_to_4d ---------------------------------------- */
/* Replaces aten._convert_weight_to_int4pack(uint8[N,K/2], inner_k_tiles)
 * (reference call: quantize_/workflows/int4/int4_tile_packed_to_4d_tensor.py:198-204).
 * in : q_u8[N][K/2], byte = q[n,2j]<<4 | q[n,2j+1];  N%8==0, K%(inner_k_tiles*16)==0
 * out: int32 [N/8][K/(inner_k_tiles*16)][32][inner_k_tiles/2]                     */
int ao_int4_pack_tile4d(const uint8_t* q_u8, int32_t* qdata, int N, int K,
                        int inner_k_tiles, void* stream);
/* HQQ qparams + 4-bit codes for a bf16 weight (the reference's int4 benchmark recipe:
 * Int4WeightOnlyConfig(int4_choose_qparams_algorithm="hqq")).  Replaces
 * _choose_qparams_and_quantize_affine_hqq + optimize_weights_proximal_legacy
 * (quantization/quant_primitives.py:1797-2002) as called at
 * quantize_/workflows/int4/int4_tile_packed_to_4d_tensor.py:149-167 (nbits 4, axis 1, raw_output False).
 * in : w bf16 [N][K] (already padded), group_size in {32,64,128,256} dividing K
 * out: q uint8 [N][K] (one code 0..15 per byte), scale / zero bf16 [N][K/group_size] in the tinygemm
 *      convention W^ = (q - 8) * scale + zero
 * workspace: device scratch of ao_int4_hqq_workspace_bytes(N, K, group_size) bytes (not shared with the linears). */
size_t ao_int4_hqq_workspace_bytes(int N, int K, int group_size);
int ao_int4_hqq_quantize(const uint16_t* w, int N, int K, int group_size, uint8_t* q, uint16_t* scale,
                         uint16_t* zero, void* workspace, size_t workspace_bytes, void* stream);
/* Inverse of the above: qdata -> q_u8[N][K/2] (used by dequantize() and tests). */
int ao_int4_unpack_tile4d(const int32_t* qdata, uint8_t* q_u8, int N, int K,
                          int inner_k_tiles, void* stream);
/* Dequantise to bf16 W^[N][K] = bf16((q-8)*s+z) (the oracle's definition of the weight). */
int ao_int4_dequant_tile4d(const int32_t* qdata, const uint16_t* scale_and_zero,
                           uint16_t* w_bf16, int N, int K, int group_size, void* stream);
/* Replaces aten._weight_int4pack_mm(x, qdata, group_size, scale_and_zero) plus the
 * bias add / slice the handler does around it
 * (int4_tile_packed_to_4d_tensor.py:243-299, hot call at :287).
 * x bf16 [M,K]; qdata int32 [N/8][K/128][32][4]; scale_and_zero bf16 [K/g][N][2];
 * bias bf16 [N_out] or NULL; y bf16 [M, N_out] with N_out <= N (row stride N_out).
 * K%1024==0 (the format pads K to 1024), N%8==0, g in {32,64,128,256}.
 * impl: 0 = auto, 1 = wgmma pipeline, 2 = CUDA-core reference-grade kernel.      */
int ao_int4_tilepacked_linear(const uint16_t* x, int M, int K, const int32_t* qdata,
                              const uint16_t* scale_and_zero, int group_size, int N,
                              const uint16_t* bias, uint16_t* y, int N_out,
                              void* workspace, size_t workspace_bytes, int impl,
                              void* stream);
/* Same with a row-strided input: row m of x starts at x + m*ldx (elements; ldx >= K, ldx % 8 == 0, x 16-byte
 * aligned), e.g. a column slice of a wider activation buffer (the output slice of a fused q|k|v projection feeding
 * the next linear without a copy).  The reference's handler makes such inputs contiguous first
 * (int4_tile_packed_to_4d_tensor.py:278-282); here the TMA descriptor carries the pitch.                      */
int ao_int4_tilepacked_linear_strided(const uint16_t* x, int ldx, int M, int K, const int32_t* qdata,
                                      const uint16_t* scale_and_zero, int group_size, int N,
                                      const uint16_t* bias, uint16_t* y, int N_out,
                                      void* workspace, size_t workspace_bytes, int impl,
                                      void* stream);
/* torch._grouped_mm(x, W.transpose(-2, -1), offs) for a 3-D Int4TilePackedTo4dTensor expert weight W [E, N_out, K],
 * 2-D x 3-D form: for offs[e-1] <= m < offs[e] (offs[-1] = 0)
 *   y[m, n] = bf16( sum_k x[m,k] * bf16((q[e][n,k]-8)*s + z) ),  n < N_out, f32 accumulate,
 * weights dequantised inside the wgmma kernel exactly as ao_int4_tilepacked_linear does.  x bf16 [M,K] (tokens sorted
 * by expert, rows contiguous); qdata int32 [E][N/8][K/128][32][4]; scale_and_zero bf16 [E][K/g][N][2]; N the padded
 * feature count (the expert stride), N_out <= N the row stride of y [M, N_out]; offs int32 [E] on the device,
 * cumulative row ends.  The host never reads offs (no sync, CUDA-graph capturable); the kernel clamps each offs[e]
 * into [offs[e-1], M].  Rows from offs[E-1] on are not written.
 * 1 <= E <= 1024, K % 1024 == 0, N % 8 == 0, g in {32,64,128,256}, no bias.                                         */
int ao_int4_tilepacked_grouped_mm(const uint16_t* x, int M, int K, const int32_t* qdata,
                                  const uint16_t* scale_and_zero, int group_size, int E, int N, int N_out,
                                  const int32_t* offs, uint16_t* y, void* workspace, size_t workspace_bytes,
                                  void* stream);
/* int8 dynamic activation x int8 weight --------------------------------------- */
/* Per-token symmetric int8 quantisation of activations: replaces
 * Int8Tensor.from_hp(x, PerRow()) on the hot path (int8_tensor.py:176-248 via
 * quantize_tensor_kwargs.py:36-71).  x bf16 [M,K] -> q int8 [M,K], scale f32 [M].  */
int ao_int8_quantize_rowwise(const uint16_t* x, int M, int K, int8_t* q, float* scale,
                             void* stream);
/* Static (calibrated) int8 quantisation of activations, one launch: replaces x * act_pre_scale followed by
 * Int8Tensor.from_hp(x, g, mapping, scale=act_quant_scale, zero_point=act_quant_zero_point) (int8_tensor.py:212-230,
 * :280-294) on CUDA tensors:
 *   q[m,k] = int8(clamp(rne(xp[m,k] * (1 / scale[m])) + zp[m], qmin, qmax)),
 * xp = x * pre_scale[k] in fp32, rounded to bf16 when pre_scale_dtype = 1 (bf16 [K]), kept in fp32 when it is 2 (f32
 * [K]); xp = x when it is 0 (pre_scale NULL).  1 / scale is the IEEE reciprocal, rne rounds half to even, a NaN gives 0.
 * scale f32 and zero_point int8 (NULL: zeros) are device memory, one value or (*_per_row != 0) one per row [M]; they
 * are never read on the host.  Outputs: q int8 [M,K] (dense), x_scale f32 [M] (the per-row scale ao_int8_dyn_linear
 * takes), x_zero_point int8 [M] (NULL: not written).  x bf16 [M][ldx] (ldx >= K, ldx % 8 == 0, 16-byte aligned),
 * pre_scale 16-byte aligned, K % 8 == 0, -128 <= qmin <= qmax <= 127.                                                */
int ao_int8_quantize_static(const uint16_t* x, int ldx, int M, int K, const void* pre_scale, int pre_scale_dtype,
                            const float* scale, int scale_per_row, const int8_t* zero_point, int zp_per_row, int qmin,
                            int qmax, int8_t* q, float* x_scale, int8_t* x_zero_point, void* stream);
/* Replaces _int_scaled_matmul + the epilogue (int8/kernels.py:114-144,
 * int8_tensor.py:305-359): y = bf16(bf16(acc_i32 * x_scale[m]) * w_scale[n] + bias[n]).
 * xq int8 [M,K] (16-byte aligned), wq int8 [N,K] (K-major, i.e. the stored qdata), scales f32.  K % 16 == 0,
 * N % 8 == 0. */
int ao_int8_dyn_linear(const int8_t* xq, const float* x_scale, int M, int K,
                       const int8_t* wq, const float* w_scale, int N,
                       const uint16_t* bias, uint16_t* y, void* workspace,
                       size_t workspace_bytes, void* stream);
/* int8 weight-only: bf16 activations on the stored int8 weights, per-row scale (a per-tensor scale expanded to
 * [N]).  Replaces torch.mm(x, qdata.t().to(bf16)) * scale.to(bf16) + bias (int8_tensor.py:336-359) with the same
 * three roundings: y = bf16(bf16(bf16(acc_f32) * bf16(w_scale[n])) + bias[n]); no add without a bias.
 * x bf16 [M][ldx] (ldx >= K, ldx % 8 == 0, 16-byte aligned), wq int8 [N,K], w_scale f32 [N]; K % 16 == 0, any N. */
int ao_int8_weight_linear(const uint16_t* x, int ldx, int M, int K, const int8_t* wq, const float* w_scale,
                          int N, const uint16_t* bias, uint16_t* y, void* workspace,
                          size_t workspace_bytes, void* stream);
/* fp8 weight-only: bf16 activations on the stored e4m3 weights, per-row scale (a per-tensor scale expanded to [N]).
 * Replaces torch.matmul(x, dequantize(W).t()) + bias (float8_tensor.py:459-469) with the same roundings: each weight
 * w~ = bf16(fp32(e4m3(wq[n,k]) * w_scale[n])), y = bf16(bf16(sum_k x[m,k] * w~[n,k]) + bias[n]); no add without a bias.
 * x bf16 [M][ldx] (ldx >= K, ldx % 8 == 0, 16-byte aligned), wq e4m3 [N,K], w_scale f32 [N] (16-byte aligned);
 * K % 16 == 0, any N. */
int ao_fp8_weight_linear(const uint16_t* x, int ldx, int M, int K, const uint8_t* wq, const float* w_scale,
                         int N, const uint16_t* bias, uint16_t* y, void* workspace,
                         size_t workspace_bytes, void* stream);
/* NF4 (QLoRA) weight-only: bf16 activations on the stored NF4Tensor of a bf16 weight [N, K].  Replaces
 * F.linear(x, W.get_original_weight()) + bias (nf4_tensor.py) with the same roundings: per flat block
 * b = (n*K + k) / block_size the scaler s[b] = bf16(bf16(quantized_scalers[b] / quantization_factor[b / scaler_block_size])
 * + scaler_mean), each weight w~ = bf16(nf4[code] * s[b]), y = bf16(bf16(sum_k x[m,k] * w~[n,k]) + bias[n]); no add
 * without a bias.  x bf16 [M][ldx] (ldx >= K, ldx % 8 == 0, 16-byte aligned); quantized_data uint8 [N*K/2] (codes of
 * the row-major weight, even element in the high nibble, 16-byte aligned); quantized_scalers int8 [N*K/block_size];
 * quantization_factor bf16 [N*K/(block_size*scaler_block_size)]; scaler_mean bf16 (one value); nf4 bf16 [16].
 * block_size % 16 == 0, K % block_size == 0, K % 32 == 0, N*K/block_size a multiple of scaler_block_size and at most
 * 2^31 - 1; any N. */
int ao_nf4_linear(const uint16_t* x, int ldx, int M, int K, const uint8_t* quantized_data,
                  const int8_t* quantized_scalers, const uint16_t* quantization_factor, const uint16_t* scaler_mean,
                  const uint16_t* nf4, int block_size, int scaler_block_size, int N, const uint16_t* bias, uint16_t* y,
                  void* workspace, size_t workspace_bytes, void* stream);
/* torch._grouped_mm(x, W.transpose(-2, -1), offs) for a 3-D weight-only Float8Tensor expert weight W [E, N, K],
 * 2-D x 3-D form (float8_tensor.py:1085-1122, weight-only branch: torch._grouped_mm on W.dequantize()): for
 * offs[e-1] <= m < offs[e] (offs[-1] = 0)
 *   y[m, n] = bf16( sum_k x[m,k] * bf16(fp32(e4m3(wq[e][n,k]) * w_scale[e][n])) ),  f32 accumulate,
 * each weight dequantized as ao_fp8_weight_linear does.  x bf16 [M,K] (tokens sorted by expert, rows contiguous,
 * 16-byte aligned); wq e4m3 [E][N][K] (the stored qdata); w_scale f32 [E][N] (16-byte aligned); offs int32 [E] on the
 * device, cumulative row ends.  The host never reads offs (no sync, CUDA-graph capturable); the kernel clamps each
 * offs[e] into [offs[e-1], M].  Rows from offs[E-1] on are not written.
 * 1 <= E <= 1024, K % 16 == 0, N % 8 == 0, no bias.                                                              */
int ao_fp8_weight_grouped_mm(const uint16_t* x, int M, int K, const uint8_t* wq, const float* w_scale, int E, int N,
                             const int32_t* offs, uint16_t* y, void* workspace, size_t workspace_bytes,
                             void* stream);
/* torch._grouped_mm(x, W.transpose(-2, -1), offs) for a 3-D weight-only Int8Tensor expert weight W [E, N, K], 2-D x 3-D
 * form, as the per-expert recipe select + ao_int8_weight_linear computes it: for offs[e-1] <= m < offs[e]
 * (offs[-1] = 0)
 *   y[m, n] = bf16( bf16(bf16(sum_k x[m,k] * wq[e][n,k]) * bf16(w_scale[e][n])) ),  f32 accumulate (exact products).
 * x bf16 [M,K] (tokens sorted by expert, rows contiguous, 16-byte aligned); wq int8 [E][N][K] (the stored qdata);
 * w_scale f32 [E][N] (a per-tensor scale expanded); offs int32 [E] on the device, cumulative row ends.  The host never
 * reads offs (no sync, CUDA-graph capturable); the kernel clamps each offs[e] into [offs[e-1], M].  Rows from
 * offs[E-1] on are not written.  1 <= E <= 1024, K % 16 == 0, any N, no bias.                                       */
int ao_int8_weight_grouped_mm(const uint16_t* x, int M, int K, const int8_t* wq, const float* w_scale, int E, int N,
                              const int32_t* offs, uint16_t* y, void* workspace, size_t workspace_bytes,
                              void* stream);
/* torch._grouped_mm(x, W.transpose(-2, -1), offs) for a 3-D Int8Tensor expert weight W [E, N, K] with symmetric
 * per-token int8 activations (dynamic PerRow, or static PerTensor after ao_int8_quantize_static), as the per-expert
 * recipe select + ao_int8_dyn_linear computes it: for offs[e-1] <= m < offs[e]
 *   y[m, n] = bf16( bf16(acc_i32[m, n] * x_scale[m]) * w_scale[e][n] ),  acc_i32 = sum_k xq[m,k] * wq[e][n,k].
 * xq int8 [M,K] (16-byte aligned), x_scale f32 [M], wq int8 [E][N][K], w_scale f32 [E][N], offs as above.
 * 1 <= E <= 1024, K % 16 == 0, N % 8 == 0, no bias.                                                                 */
int ao_int8_dyn_grouped_mm(const int8_t* xq, const float* x_scale, int M, int K, const int8_t* wq,
                           const float* w_scale, int E, int N, const int32_t* offs, uint16_t* y, void* workspace,
                           size_t workspace_bytes, void* stream);
/* int32 accumulator only (aten._int_mm equivalent; int8/kernels.py:18-76).  xq 16-byte aligned, K % 16 == 0. */
int ao_int8_mm_i32(const int8_t* xq, int M, int K, const int8_t* wq, int N, int32_t* acc,
                   void* workspace, size_t workspace_bytes, void* stream);

/* fp8 e4m3 rowwise -------------------------------------------------------------- */
/* Replaces _choose_scale_float8 + _quantize_affine_float8 for PerRow activations
 * (quant_primitives.py:2172-2287, float8_tensor.py:235-242).
 * x bf16 [M,K] -> q e4m3 [M,K] (bytes), scale f32 [M] = f32(bf16(amax/448)).          */
int ao_fp8_quantize_rowwise(const uint16_t* x, int M, int K, uint8_t* q, float* scale,
                            void* stream);
/* Replaces torch._scaled_mm(a, b, scale_a, scale_b, bias, out_dtype=bf16)
 * (float8/inference.py:86-123 <- float8_tensor.py:449-457).
 * y = bf16( (Xq Wq^T)[m,n] * x_scale[m] * w_scale[n] + bias[n] ), f32 accumulate.
 * xq 16-byte aligned, K % 16 == 0, N % 16 == 0.                                       */
int ao_fp8_rowwise_linear(const uint8_t* xq, const float* x_scale, int M, int K,
                          const uint8_t* wq, const float* w_scale, int N,
                          const uint16_t* bias, uint16_t* y, void* workspace,
                          size_t workspace_bytes, void* stream);
/* Static (calibrated) e4m3 quantisation of activations, one launch: replaces PrototypeFloat8Tensor.from_hp(x,
 * scale=act_quant_scale) (prototype_float8_tensor.py:182-203, quant_primitives.py:2271-2287) on CUDA tensors:
 *   q[m,k] = e4m3(clamp(fp32(x[m,k]) / scale[m], -448, 448)),
 * an IEEE division (not a reciprocal multiply); a NaN quotient stays NaN, x / 0 = +-inf gives +-448, 0 / 0 NaN.
 * scale f32 is device memory, one value or (scale_per_row != 0) one per row [M]; it is never read on the host.
 * Outputs: q e4m3 [M,K] (dense bytes), x_scale f32 [M] (the per-row scale ao_fp8_rowwise_linear takes).
 * x bf16 [M][ldx] (ldx >= K, ldx % 8 == 0, 16-byte aligned), K % 8 == 0.                                           */
int ao_fp8_quantize_static(const uint16_t* x, int ldx, int M, int K, const float* scale, int scale_per_row, uint8_t* q,
                           float* x_scale, void* stream);
/* The linear of PrototypeFloat8Tensor (prototype_float8_tensor.py:329-474) on the codes of ao_fp8_quantize_static:
 *   y[m,n] = bf16( (Xq Wq^T)[m,n] * (x_scale[m] * w_scale[n]) + bias[n] ),
 * as ao_fp8_rowwise_linear computes it, with w_scale[0] for every n when w_scale_per_row == 0 (a PerTensor weight:
 * no [N] copy of its scale).  With out_scale (NULL: none), the output fake-quant (output_act_quant_scale, :461-472)
 * follows in the GEMM's epilogue:
 *   out[m,n] = bf16(fp32(e4m3(clamp(fp32(y[m,n]) / s, -448, 448))) * s),
 * s = out_scale[0], or out_scale[m] when out_scale_per_row != 0 (device memory, never read on the host); the division
 * is IEEE, as in ao_fp8_quantize_static.  xq 16-byte aligned, K % 16 == 0, N % 16 == 0.                             */
int ao_fp8_static_linear(const uint8_t* xq, const float* x_scale, int M, int K, const uint8_t* wq, const float* w_scale,
                         int w_scale_per_row, int N, const uint16_t* bias, const float* out_scale, int out_scale_per_row,
                         uint16_t* y, void* workspace, size_t workspace_bytes, void* stream);
/* Replaces torchao's aten._grouped_mm handler for a rowwise Float8Tensor expert weight, i.e.
 * torch._scaled_grouped_mm / F.scaled_grouped_mm rowwise (float8_tensor.py:1085-1122), 2-D x 3-D form:
 * for offs[e-1] <= m < offs[e] (offs[-1] = 0):
 *   y[m, :] = bf16( (Xq[m] Wq[e]^T) * x_scale[m] * w_scale[e, :] ), f32 accumulate.
 * xq e4m3 [M,K] (tokens sorted by expert, 16-byte aligned); wq e4m3 [E][N][K] (K-major, the stored qdata);
 * x_scale f32 [M]; w_scale f32 [E][N]; offs int32 [E] on the device, cumulative row ends.  The host never reads offs
 * (no sync, CUDA-graph capturable); the kernel clamps each offs[e] into [offs[e-1], M].  Rows from offs[E-1] on are
 * not written.  1 <= E <= 1024, K % 16 == 0, N % 16 == 0, no bias.                                             */
int ao_fp8_rowwise_grouped_mm(const uint8_t* xq, const float* x_scale, int M, int K,
                              const uint8_t* wq, const float* w_scale, int E, int N,
                              const int32_t* offs, uint16_t* y, void* workspace,
                              size_t workspace_bytes, void* stream);
/* Replaces torch.bmm(x, w) on a [B, K, N] rowwise Float8Tensor (float8_tensor.py:472-522, mslk's
 * f8f8bf16_rowwise_batched on a transposed copy): xq e4m3 [B*M, K] with x_scale [B*M] (per row), batch b's weights
 * with w_scale [B, N]: y bf16 [B*M, N] = bf16(acc * x_scale[m] * w_scale[b, n]), no bias term.  w_kn = 0: wq is stored
 * [B, N, K] (w is its transposed view); w_kn = 1: wq is stored [B, K, N], read as it is (no transposed copy).
 * Two launches: the row ends (b + 1) * M written into the workspace on the device, then the grouped GEMM.
 * 1 <= B <= 1024, K % 16 == 0, N % 16 == 0.  At M == 0 it returns before reading any pointer. */
int ao_fp8_rowwise_bmm(const uint8_t* xq, const float* x_scale, int B, int M, int K, const uint8_t* wq,
                       const float* w_scale, int N, int w_kn, uint16_t* y, void* workspace, size_t workspace_bytes,
                       void* stream);

/* fp8 e4m3 blockwise: 1x128 activation blocks, 128x128 weight blocks -------------- */
/* Replaces Float8Tensor.from_hp(x, PerBlock([1, 128])) for activations (_choose_scale_float8 +
 * _quantize_affine_float8, quant_primitives.py:2173-2212, :2271-2287): per block of 128 elements of a row,
 * s = f32(bf16(amax/448)) and q = e4m3(clamp(f32(x)/s, -448, 448)); NaN propagates as in torch.amax / torch.clamp, and
 * an all-zero block has s = 0 and NaN codes (0/0).  x bf16 [M,K] -> q e4m3 [M,K] (the reference's codes) and the
 * scales TRANSPOSED, scale_t f32 [K/128][ldm] with ldm = M rounded up to a multiple of 4 (the layout the GEMM loads;
 * scale_t[kb][m] is the reference's scale[m][kb]; the pad entries m >= M are written as 0).  K % 128 == 0. */
int ao_fp8_quantize_1x128(const uint16_t* x, int M, int K, uint8_t* q, float* scale_t, void* stream);
/* The same with row pitch ldx (elements; ldx >= K, ldx % 8 == 0, x 16-byte aligned), see the _ld variants below. */
int ao_fp8_quantize_1x128_ld(const uint16_t* x, int ldx, int M, int K, uint8_t* q, float* scale_t, void* stream);
/* Replaces the reference's blockwise GEMM (its Triton loop, float8/kernels.py:86-97, called from
 * float8_tensor.py:431-447):
 *   acc[m,n] = sum over 128-k blocks kb, in order, of (Xq Wq^T)_kb[m,n] * x_scale[m][kb] * w_scale[n/128][kb]  (f32)
 *   y = bf16(bf16(acc) + bias[n]); no add without a bias.
 * Each block's product and scale multiply-add are one fp32 fma on the block's partial times x_scale.
 * xq e4m3 [M,K] (16-byte aligned); x_scale_t f32 [K/128][round_up(M,4)] as ao_fp8_quantize_1x128 writes it (16-byte
 * aligned); wq e4m3 [N,K]; w_scale f32 [N/128][K/128].  K % 128 == 0, N % 128 == 0. */
int ao_fp8_blockwise_linear(const uint8_t* xq, const float* x_scale_t, int M, int K, const uint8_t* wq,
                            const float* w_scale, int N, const uint16_t* bias, uint16_t* y, void* workspace,
                            size_t workspace_bytes, void* stream);
/* F.linear(x, Float8Sparse2x4_2DData2DMetadataTensor): 2:4-sparse e4m3 weights with per-row scales and per-token
 * e4m3 activations, as the reference's CUTLASS sparse GEMM computes it:
 *   acc[m,n] = sum_k xq[m,k] * W[n,k]   (W the decompressed codes; no per-chunk promotion)
 *   y[m,n] = bf16(fma(acc[m,n] * w_scale[n], x_scale[m], bias[n]))   (fp32; bias 0 if null)
 * xq e4m3 [M,K] (16-byte aligned); x_scale f32 [M]; wq e4m3 [N][K/2], the two kept codes of each 4-k group (16-byte
 * aligned); w_meta uint8, round_up(N,64) x round_up(K,128)/8 bytes in CUTLASS's Sm90 8-bit metadata layout (16-byte
 * aligned); w_scale f32 [N].  K % 32 == 0, N % 16 == 0.  Metadata of rows >= N or k >= K is never used, and an
 * all-zero group's nibble (0b0000) is fed as 0b0100.  At M == 0 it returns before reading any pointer. */
int ao_fp8_sparse_linear(const uint8_t* xq, const float* x_scale, int M, int K, const uint8_t* wq, const uint8_t* w_meta,
                         const float* w_scale, int N, const uint16_t* bias, uint16_t* y, void* workspace,
                         size_t workspace_bytes, void* stream);
/* torch._grouped_mm(x, W.transpose(-2, -1), offs) for a 3-D blockwise Float8Tensor expert weight W [E, N, K]
 * (block_size [1, 128, 128]), 2-D x 3-D form, as the per-expert recipe select + ao_fp8_blockwise_linear computes it:
 * for offs[e-1] <= m < offs[e] (offs[-1] = 0)
 *   acc[m,n] = sum over 128-k blocks kb, in order, of (Xq Wq[e]^T)_kb[m,n] * x_scale[m][kb] * w_scale[e][n/128][kb]
 *   y[m,n] = bf16(acc[m,n]),  no bias.
 * xq e4m3 [M,K] (tokens sorted by expert, 16-byte aligned); x_scale_t f32 [K/128][round_up(M,4)] as
 * ao_fp8_quantize_1x128 writes it over all M rows (16-byte aligned); wq e4m3 [E][N][K] (the stored qdata); w_scale f32
 * [E][N/128][K/128]; offs int32 [E] on the device, cumulative row ends.  The host never reads offs (no sync,
 * CUDA-graph capturable); the kernel clamps each offs[e] into [offs[e-1], M].  Rows from offs[E-1] on are not written.
 * 1 <= E <= 1024, K % 128 == 0, N % 128 == 0.  At M == 0 it returns before reading any pointer. */
int ao_fp8_blockwise_grouped_mm(const uint8_t* xq, const float* x_scale_t, int M, int K, const uint8_t* wq,
                                const float* w_scale, int E, int N, const int32_t* offs, uint16_t* y, void* workspace,
                                size_t workspace_bytes, void* stream);

/* mxfp8 (e4m3 data, e8m0 block-32 scales) --------------------------------------- */
/* Replaces MXTensor.to_mx(x, e4m3, 32, RCEIL, is_swizzled_scales) for activations
 * (mx_tensor.py:228-409, :161-225).  x bf16 [M,K] -> q e4m3 [M,K], scales e8m0 bytes;
 * swizzled=1 writes the 128x4 -> 32x16 blocked layout (mx_formats/utils.py:31-70),
 * size 32*ceil(M/128) x 16*ceil(K/128); swizzled=0 writes plain [M][K/32].            */
int ao_mxfp8_quantize(const uint16_t* x, int M, int K, uint8_t* q, uint8_t* scale_e8m0,
                      int swizzled, void* stream);
/* Replaces torch._scaled_mm(e4m3, e4m3, e8m0 blocked, e8m0 blocked, bias, bf16)
 * (mx_tensor.py:803-810).  Both scale tensors are in the blocked layout.  xq 16-byte aligned,
 * K % 32 == 0.                                                                        */
int ao_mxfp8_linear(const uint8_t* xq, const uint8_t* x_scale_blocked, int M, int K,
                    const uint8_t* wq, const uint8_t* w_scale_blocked, int N,
                    const uint16_t* bias, uint16_t* y, void* workspace,
                    size_t workspace_bytes, void* stream);

/* mxfp4 (e2m1 data, e8m0 block-32 scales) --------------------------------------- */
/* Replaces MXTensor.to_mx(x, float4_e2m1fn_x2, 32, RCEIL, is_swizzled_scales) for activations
 * (mx_tensor.py:228-409, :161-225): per 32-element block e8 = rceil(amax * f32(1/6)) (0xFF for inf / NaN),
 * codes e2m1(x * 2^(127-e8)) rounded to nearest even and saturated at 6.  x bf16 [M,K] -> q uint8 [M,K/2]
 * (even k in the LOW nibble), scales e8m0 bytes, plain [M][K/32] or (swizzled=1) blocked as for mxfp8 with the
 * padding written as zero.  K % 32 == 0.                                                                     */
int ao_mxfp4_quantize(const uint16_t* x, int M, int K, uint8_t* q, uint8_t* scale_e8m0,
                      int swizzled, void* stream);
/* y = bf16( sum_k xhat[m,k] * what[n,k] (fp32) + bias ), xhat / what = each operand's code x 2^(e8-127), the
 * MXTensor.dequantize() of both (exact in bf16 for every scale byte: the products of the block-scaled fp4 MMA).
 * xq uint8 [M,K/2] (16-byte aligned), wq uint8 [N,K/2], both scale tensors in the blocked layout with zero padding.  K % 32 == 0
 * (a K tail of the last 128-k chunk is zero-filled), any N.                                                  */
int ao_mxfp4_linear(const uint8_t* xq, const uint8_t* x_scale_blocked, int M, int K,
                    const uint8_t* wq, const uint8_t* w_scale_blocked, int N,
                    const uint16_t* bias, uint16_t* y, void* workspace,
                    size_t workspace_bytes, void* stream);

/* nvfp4 (e2m1 data, e4m3 block-16 scales, f32 per-tensor scale) ------------------ */
/* Replaces nvfp4_quantize + to_blocked for activations (nvfp4_tensor.py:772-854).
 * x bf16 [M,K] -> q uint8 [M,K/2] (even k in the LOW nibble), scales e4m3 bytes.
 * per_tensor_scale: device f32 scalar or NULL (single-level scaling).                 */
int ao_nvfp4_quantize(const uint16_t* x, int M, int K, const float* per_tensor_scale,
                      uint8_t* q, uint8_t* scale_e4m3, int swizzled, void* stream);
/* Replaces torch._scaled_mm(fp4x2, fp4x2, e4m3 blocked scales) * (a_pts*b_pts) + bias
 * (nvfp4_tensor.py:487-578).  a_pts / b_pts: device f32 scalars or NULL (=1).  xq 16-byte aligned,
 * K % 256 == 0, N % 16 == 0.                                                          */
int ao_nvfp4_linear(const uint8_t* xq, const uint8_t* x_scale_blocked, const float* a_pts,
                    int M, int K, const uint8_t* wq, const uint8_t* w_scale_blocked,
                    const float* b_pts, int N, const uint16_t* bias, uint16_t* y,
                    void* workspace, size_t workspace_bytes, void* stream);
/* nvfp4 weight-only and nvfp4-weight x fp8-rowwise-activation (BASELINE config 5):
 * y = bf16( (sum_k x[m,k] * e2m1(W)[n,k] * blockscale[n,k/16]) * x_scale[m] * b_pts + bias ),
 * weights dequantised to bf16 inside the wgmma kernel.  x is bf16 [M,K]; x_scale f32 [M] or NULL.
 * Semantics = F.linear(x_dq, NVFP4Tensor.dequantize()) (nvfp4_tensor.py:199-231,
 * inference_workflow.py:356-400); for e4m3 activations pass the output of ao_fp8_fakequant_rowwise. */
int ao_nvfp4_weight_linear(const uint16_t* x, const float* x_scale, int M, int K,
                           const uint8_t* wq, const uint8_t* w_scale_blocked,
                           const float* b_pts, int N, const uint16_t* bias, uint16_t* y,
                           void* workspace, size_t workspace_bytes, void* stream);
/* Same with (a) a row-strided input (row m of x at x + m*ldx elements, ldx >= K, ldx % 8 == 0: e.g. a column slice
 * of a fused projection's output) and (b) b_pts_per_row != 0: b_pts is one f32 scale PER OUTPUT FEATURE [N] instead of
 * a scalar -- a fused q|k|v or gate|up group of NVFP4 weights keeps each member's own per-tensor scale
 * (ao_b200/fusion.py; the reference has one scalar per NVFP4Tensor, nvfp4_tensor.py:69-79).                      */
int ao_nvfp4_weight_linear_ex(const uint16_t* x, int ldx, const float* x_scale, int M, int K,
                              const uint8_t* wq, const uint8_t* w_scale_blocked, const float* b_pts,
                              int b_pts_per_row, int N, const uint16_t* bias, uint16_t* y,
                              void* workspace, size_t workspace_bytes, void* stream);
/* Replaces torchao's aten._grouped_mm handler for an NVFP4Tensor expert weight (nvfp4_tensor.py:709-753), 2-D x 3-D
 * form: for offs[e-1] <= m < offs[e] (offs[-1] = 0)
 *   y[m, :] = bf16( (sum_k x[m,k] * e2m1(Wq[e])[:,k] * blockscale[e][:,k/16]) * x_scale[m] * w_pts[e] ),
 * weights dequantised exactly inside the wgmma kernel.  x bf16 [M,K] (tokens sorted by expert; for NVFP4 activations
 * the xhat of ao_nvfp4_fakequant_grouped); x_scale f32 [M] or NULL; wq uint8 [E][N][K/2] (the stored qdata);
 * w_scale_blocked: each expert's [N, K/16] e4m3 scales in the blocked layout, one after the other; w_pts f32 [E];
 * offs int32 [E] on the device, cumulative row ends.  The host never reads offs (no sync, CUDA-graph capturable); the
 * kernel clamps each offs[e] into [offs[e-1], M].  Rows from offs[E-1] on are not written.
 * 1 <= E <= 1024, K % 128 == 0, N % 128 == 0, no bias.                                                              */
int ao_nvfp4_grouped_mm(const uint16_t* x, const float* x_scale, int M, int K, const uint8_t* wq,
                        const uint8_t* w_scale_blocked, const float* w_pts, int E, int N,
                        const int32_t* offs, uint16_t* y, void* workspace, size_t workspace_bytes, void* stream);
/* The activations of the above, each expert's rows quantized to NVFP4 with that expert's own per-tensor scale
 * a_pts[e] = amax(|x[rows of e]|) / (448 * 6), exactly as ao_nvfp4_quantize(x[rows of e], a_pts[e]) quantizes them,
 * the rows of e being [end[e-1], end[e]) with end[e] = min(M, max(0, offs[0..e])) as in the GEMM.
 * xhat bf16 [M,K] = each element's e2m1 code times its e4m3 block scale (exact in bf16); x_scale f32 [M] = a_pts of
 * the row's expert.  An all-zero expert and the rows past end[E-1] get xhat = 0 and x_scale = 0.  x has row pitch ldx
 * (elements; ldx >= K, ldx % 8 == 0, x 16-byte aligned); row_amax: f32 [M] device scratch.  K % 16 == 0, E >= 1.
 * Two kernels; offs is never read on the host.                                                                      */
int ao_nvfp4_fakequant_grouped(const uint16_t* x, int ldx, int M, int K, const int32_t* offs, int E,
                               uint16_t* xhat, float* x_scale, float* row_amax, void* stream);
/* torch._grouped_mm(x, W.transpose(-2, -1), offs) for a 3-D MXTensor expert weight W [E, N, K] (mxfp8 / mxfp4), 2-D x
 * 3-D form, as the per-expert recipe select + ao_mx*_linear computes it: for offs[e-1] <= m < offs[e] (offs[-1] = 0)
 *   y[m, :] = bf16( sum_k x[m,k] * what[e][:,k] ),  f32 accumulate, what = code x 2^(e8 - 127) dequantised exactly
 * inside the wgmma kernel.  x bf16 [M,K] (tokens sorted by expert, rows contiguous, 16-byte aligned: the xhat of
 * ao_mx*_fakequant); wq [E][N][K] e4m3 (mxfp8) or [E][N][K/2] packed e2m1, even k in the low nibble (mxfp4);
 * w_scale_blocked: the blocked e8m0 scales of the [E*N, K/32] scales (each expert's blocked scales one after the
 * other); offs int32 [E] on the device, cumulative row ends.  The host never reads offs (no sync, CUDA-graph
 * capturable); the kernel clamps each offs[e] into [offs[e-1], M].  Rows from offs[E-1] on are not written.
 * 1 <= E <= 1024, K % 32 == 0, N % 128 == 0, no bias.                                                              */
int ao_mxfp8_grouped_mm(const uint16_t* x, int M, int K, const uint8_t* wq, const uint8_t* w_scale_blocked, int E,
                        int N, const int32_t* offs, uint16_t* y, void* workspace, size_t workspace_bytes, void* stream);
int ao_mxfp4_grouped_mm(const uint16_t* x, int M, int K, const uint8_t* wq, const uint8_t* w_scale_blocked, int E,
                        int N, const int32_t* offs, uint16_t* y, void* workspace, size_t workspace_bytes, void* stream);
/* The activations of the above: every row of x quantized as ao_mx*_quantize quantizes it (RCEIL e8m0 per 32-element
 * block) and written back as xhat bf16 [M,K] = code x 2^(e8 - 127), bit for bit what the dense MX linear dequantises
 * its activations to.  offs is not needed: MX scales couple no rows.  x bf16 [M][ldx] (ldx >= K, ldx % 8 == 0, 16-byte
 * aligned), K % 32 == 0.  One kernel.                                                                               */
int ao_mxfp8_fakequant(const uint16_t* x, int ldx, int M, int K, uint16_t* xhat, void* stream);
int ao_mxfp4_fakequant(const uint16_t* x, int ldx, int M, int K, uint16_t* xhat, void* stream);
/* Per-token e4m3 quantisation that keeps the codes as bf16 values (exact): xq = bf16(e4m3(x/s)),
 * s = f32(bf16(amax/448)) -- the codes of ao_fp8_quantize_rowwise, i.e. the values Float8Tensor.from_hp(x, PerRow())
 * stores (quant_primitives.py:2172-2287), in the operand type the bf16 MMA consumes.  An all-zero row (s = 0) gives
 * zeros where the e4m3 codes are NaN (0/0). */
int ao_fp8_fakequant_rowwise(const uint16_t* x, int M, int K, uint16_t* xq_bf16, float* scale,
                             void* stream);

/* Row-strided variants of the activation quantizers: row m of x starts at x + m*ldx (elements; ldx >= K,
 * ldx % 8 == 0, x 16-byte aligned) -- the input is a column slice of a wider buffer, e.g. the q part of a fused
 * q|k|v projection's output.  The reference makes such inputs contiguous with a copy kernel first; here the pitch
 * is a kernel argument.  Outputs are dense, exactly as in the functions without the suffix.                      */
int ao_int8_quantize_rowwise_ld(const uint16_t* x, int ldx, int M, int K, int8_t* q, float* scale, void* stream);
int ao_fp8_quantize_rowwise_ld(const uint16_t* x, int ldx, int M, int K, uint8_t* q, float* scale, void* stream);
int ao_mxfp8_quantize_ld(const uint16_t* x, int ldx, int M, int K, uint8_t* q, uint8_t* scale_e8m0,
                         int swizzled, void* stream);
int ao_mxfp4_quantize_ld(const uint16_t* x, int ldx, int M, int K, uint8_t* q, uint8_t* scale_e8m0,
                         int swizzled, void* stream);
int ao_nvfp4_quantize_ld(const uint16_t* x, int ldx, int M, int K, const float* per_tensor_scale,
                         uint8_t* q, uint8_t* scale_e4m3, int swizzled, void* stream);
int ao_fp8_fakequant_rowwise_ld(const uint16_t* x, int ldx, int M, int K, uint16_t* xq_bf16, float* scale,
                                void* stream);

/* Producer-fused per-token quantizers (SURVEY section 8f-1: "fused with the preceding RMSNorm / SiLU where possible").
 * They replace, for a dynamic-activation linear that follows an RMSNorm or a SiLU-gated product, the norm / activation
 * kernel(s) + Int8Tensor.from_hp(x, PerRow()) / Float8Tensor.from_hp(x, PerRow()) (int8_tensor.py:176-248,
 * float8_tensor.py:235-242) by one kernel; the scales and codes are those ao_int8/fp8_quantize_rowwise give for the
 * bf16 values the producer would have written (HF LlamaRMSNorm / LlamaMLP rounding points).  fmt: 0 int8, 1 e4m3.     */
int ao_rmsnorm_quantize_rowwise(const uint16_t* x, int ldx, const uint16_t* weight, float eps, int M, int K,
                                int fmt, uint8_t* q, float* scale, void* stream);
int ao_silu_mul_quantize_rowwise(const uint16_t* gate, int ldg, const uint16_t* up, int ldu, int M, int K,
                                 int fmt, uint8_t* q, float* scale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* AO_B200_H_ */
