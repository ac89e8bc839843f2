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
 *     must not be shared by linears running concurrently on different streams.
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
/* int8 dynamic activation x int8 weight --------------------------------------- */
/* Per-token symmetric int8 quantisation of activations: replaces
 * Int8Tensor.from_hp(x, PerRow()) on the hot path (int8_tensor.py:176-248 via
 * quantize_tensor_kwargs.py:36-71).  x bf16 [M,K] -> q int8 [M,K], scale f32 [M].  */
int ao_int8_quantize_rowwise(const uint16_t* x, int M, int K, int8_t* q, float* scale,
                             void* stream);
/* Replaces _int_scaled_matmul + the epilogue (int8/kernels.py:114-144,
 * int8_tensor.py:305-359): y = bf16(bf16(acc_i32 * x_scale[m]) * w_scale[n] + bias[n]).
 * xq int8 [M,K], wq int8 [N,K] (K-major, i.e. the stored qdata), scales f32.         */
int ao_int8_dyn_linear(const int8_t* xq, const float* x_scale, int M, int K,
                       const int8_t* wq, const float* w_scale, int N,
                       const uint16_t* bias, uint16_t* y, void* workspace,
                       size_t workspace_bytes, void* stream);
/* int32 accumulator only (aten._int_mm equivalent; int8/kernels.py:18-76). */
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
 * y = bf16( (Xq Wq^T)[m,n] * x_scale[m] * w_scale[n] + bias[n] ), f32 accumulate.     */
int ao_fp8_rowwise_linear(const uint8_t* xq, const float* x_scale, int M, int K,
                          const uint8_t* wq, const float* w_scale, int N,
                          const uint16_t* bias, uint16_t* y, void* workspace,
                          size_t workspace_bytes, void* stream);
/* Replaces torchao's aten._grouped_mm handler for a rowwise Float8Tensor expert weight, i.e.
 * torch._scaled_grouped_mm / F.scaled_grouped_mm rowwise (float8_tensor.py:1085-1122), 2-D x 3-D form:
 * for offs[e-1] <= m < offs[e] (offs[-1] = 0):
 *   y[m, :] = bf16( (Xq[m] Wq[e]^T) * x_scale[m] * w_scale[e, :] ), f32 accumulate.
 * xq e4m3 [M,K] (tokens sorted by expert); wq e4m3 [E][N][K] (K-major, the stored qdata); x_scale f32 [M];
 * w_scale f32 [E][N]; offs int32 [E] on the device, cumulative row ends.  The host never reads offs (no sync,
 * CUDA-graph capturable); the kernel clamps each offs[e] into [offs[e-1], M].  Rows from offs[E-1] on are not
 * written.  1 <= E <= 1024, K % 16 == 0, N % 16 == 0, no bias.                                             */
int ao_fp8_rowwise_grouped_mm(const uint8_t* xq, const float* x_scale, int M, int K,
                              const uint8_t* wq, const float* w_scale, int E, int N,
                              const int32_t* offs, uint16_t* y, void* workspace,
                              size_t workspace_bytes, void* stream);

/* mxfp8 (e4m3 data, e8m0 block-32 scales) --------------------------------------- */
/* Replaces MXTensor.to_mx(x, e4m3, 32, RCEIL, is_swizzled_scales) for activations
 * (mx_tensor.py:228-409, :161-225).  x bf16 [M,K] -> q e4m3 [M,K], scales e8m0 bytes;
 * swizzled=1 writes the 128x4 -> 32x16 blocked layout (mx_formats/utils.py:31-70),
 * size 32*ceil(M/128) x 16*ceil(K/128); swizzled=0 writes plain [M][K/32].            */
int ao_mxfp8_quantize(const uint16_t* x, int M, int K, uint8_t* q, uint8_t* scale_e8m0,
                      int swizzled, void* stream);
/* Replaces torch._scaled_mm(e4m3, e4m3, e8m0 blocked, e8m0 blocked, bias, bf16)
 * (mx_tensor.py:803-810).  Both scale tensors are in the blocked layout.              */
int ao_mxfp8_linear(const uint8_t* xq, const uint8_t* x_scale_blocked, int M, int K,
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
 * (nvfp4_tensor.py:487-578).  a_pts / b_pts: device f32 scalars or NULL (=1).          */
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
