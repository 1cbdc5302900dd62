/* uav_b200_int8.h — C ABI of libuav_b200.so for the LLaVA captioner's weight-only int8 (W8A16) decoder Linears.
 * Conventions as in uav_b200.h: raw device pointers, explicit shapes, caller-owned memory, stream-ordered calls that
 * never synchronise, a uav_status_t per call and uav_last_error_string() on failure.
 *
 * Weight format: an int8 matrix q [N][K] (row-major, dense) with an fp32 per-row absmax[N].  Row n holds
 *   absmax[n] = max_k |w[n][k]|                       (fp32, from the fp16 weights)
 *   q[n][k]   = round_half_even((w[n][k] * 127) / absmax[n])    (IEEE fp32 division; a row with absmax 0 is all 0)
 * which is bitsandbytes' row-wise int8 rule.  Decode uses the weight q * absmax / 127 exactly (the GEMV scales its
 * fp32 sum once per output); the prefill dequantizes to fp16((q * absmax) / 127), one more rounding per weight.
 */
#ifndef UAV_B200_INT8_H_
#define UAV_B200_INT8_H_

#include "uav_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* quantizes fp16 w [N][K] (row stride ldw elements) into q [N][K] int8 and absmax [N] fp32 with the rule above; one
 * warp per row.  q and absmax may point at a row slice of a larger matrix (a fused q|k|v or gate|up filled one
 * released tensor at a time).  K % 16 == 0, ldw % 8 == 0, w and q 16-byte aligned. */
uav_status_t uav_quantize_rows_int8(const void* w, int64_t N, int64_t K, int64_t ldw, void* q, float* absmax,
                                    uav_stream_t stream);
/* out[n][k] = fp16((q[n][k] * absmax[n]) / 127), fp16 [N][K] dense, for the prefill GEMMs.  K % 16 == 0, q and out
 * 16-byte aligned. */
uav_status_t uav_dequantize_rows_int8(const void* q, const float* absmax, int64_t N, int64_t K, void* out,
                                      uav_stream_t stream);
/* the int8 decode weight stream on 1 <= rows <= 8 input rows: out[r][n] = (sum_k q[n][k] x[r][k]) * (absmax[n] / 127)
 * (+ residual[r][n], one rounding), fp32 accumulation; x fp16 [rows][K], residual fp16 [rows][N], out [rows][N]
 * dense, out_dtype UAV_F16 (residual or NULL) or UAV_F32 (no residual).  K % 16 == 0, K <= 16384, rows * K <= 110592
 * (x is held in shared memory); q and x 16-byte aligned.  The weights go through fp16 tensor-core MMAs with the rows
 * as the MMA's columns, one kernel for every row count and a fixed-order split-K combine: results are deterministic
 * and a row's result is bit-identical whatever the other rows of its call are. */
uav_status_t uav_gemv_rows_int8(const void* q, const float* absmax, int64_t N, int64_t K, const void* x, int64_t rows,
                                const void* residual, void* out, int out_dtype, uav_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* UAV_B200_INT8_H_ */
