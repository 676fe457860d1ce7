// Host entry points of the kernel translation units: paro_capi.cu calls them, some call each other (the pre-pass of
// paro_rotate.cu serves paro_decode.cu, paro_gemm.cu and paro_moe_grouped.cu).  Every defining file includes this header too, so
// each definition is checked against its one declaration.
#pragma once

#include <cuda_runtime.h>

#include "paro_layout.h"
#include "paro_stream.h"

namespace paro {

// paro_rotate.cu
int rotate_launch(const void *x, void *out, const int16_t *idx, const void *theta, int theta_dtype, const void *scales,
                  int scales_dtype, int64_t M, int K, int krot, int G, int dtype, cudaStream_t stream);
int rotate_backward_launch(const void *y, const void *gout, const void *x, const int16_t *idx, const void *theta, int theta_dtype, const void *scales,
                           int scales_dtype, void *grad_x, float *grad_theta, float *grad_scale, int64_t M, int K, int krot, int G, int dtype,
                           int ref_formula, cudaStream_t stream);
int rotate_backward_debug_plan(int64_t M, int K, int krot, int G, int ref_formula, int sms, int64_t *out);
int rotate_routed_launch(const Layout &L, const void *packed, bool silu_mul, const void *src, const int32_t *rows, const int32_t *live_tiles,
                         int top_k, void *out, int rows_max, int nt, cudaStream_t stream);
// the pre-pass of the tensor-core kernels: x rotated for every partition of L, M_store rows per partition (rows >= M zero) in the
// B-operand order of tiles of nt tokens, after a chain step's x op (PARO_XOP_*): NONE reads x [M, K]; SILU_MUL x [M, 2K] (gate | up);
// RMSNORM h = x [M, K] with norm_w [K] and the producing step's fp32 sums of h^2, stats[b * M + m] for its 128-column blocks b < stats_blocks
int rotate_chain_launch(const Layout &L, const void *packed, int x_op, const void *x, const void *norm_w, const float *stats, int stats_blocks,
                        float eps, void *out, int64_t M, int64_t M_store, int nt, cudaStream_t stream);

// paro_prepack.cu
int prepack_launch(const paro_linear_shape &s, const Layout &L, const int32_t *qweight, const int32_t *qzeros,
                   const void *scales, int scales_dtype, const int16_t *pairs, const void *theta, int theta_dtype,
                   const void *cscales, int cs_dtype, void *packed, cudaStream_t stream);
int unpack_dense_launch(const paro_linear_shape &s, const Layout &L, const void *packed, void *W, cudaStream_t stream);

// paro_decode.cu
bool decode_supported(const Layout &L, int64_t M);
int decode_forward(const paro_linear_shape &s, const Layout &L, const void *packed, const void *x, int64_t M,
                   const void *bias, void *y, void *scratch, size_t scratch_bytes, cudaStream_t stream);
size_t decode_scratch_bytes(const Layout &L, int64_t max_m);
int decode_trace_read(unsigned long long *host, int max_ctas);
int decode_debug_plan(const Layout &L, int64_t M, int sets, int sms, const int32_t *resident4, int32_t *out20);

// paro_stream.cu
bool stream_supported(const Layout &L, int64_t M);
size_t stream_sync_bytes(const Layout &L);
size_t stream_workspace_bytes(const Layout &L, int64_t max_m);
size_t stream_chain_workspace_bytes(const HostStep *steps, int n, int64_t M);
int stream_forward(const HostStep *steps, int n, int64_t M, void *workspace, size_t workspace_bytes, cudaStream_t stream);
int stream_trace_read(unsigned long long *host, int max_ctas);
int stream_debug_plan(const Layout &L, int64_t M, int sets, int ctas, int32_t *out);

// paro_gemm.cu
size_t gemm_workspace_bytes(const Layout &L, int64_t max_m);
int gemm_debug_plan(const Layout &L, int64_t M, int sms, int32_t *out);
int gemm_grouped_launch(const Layout &L, const void *packed, long long expert_stride, const void *xr, void *y, int NT, int slots,
                        const int32_t *rows, const int32_t *tile_expert, const int32_t *live_tiles, int dtype, cudaStream_t stream);
// a chain for any M (paro_prefill_chain_forward): per step the pre-pass with the step's x op, then the GEMM with its epilogue
size_t prefill_chain_workspace_bytes(const HostStep *steps, int n, int64_t M);
int prefill_chain_forward(const HostStep *steps, int n, int64_t M, void *workspace, size_t workspace_bytes, cudaStream_t stream);

// paro_moe.cu
size_t moe_workspace_bytes(const paro_moe_desc *d, int64_t T, int32_t k);
int moe_forward(const paro_moe_desc *d, const void *x, const int32_t *ids, const float *wts, int64_t T, int32_t k, void *h, void *y,
                void *workspace, size_t workspace_bytes, cudaStream_t stream);
int moe_debug_plan(const paro_moe_desc *d, int64_t T, int32_t k, int32_t sms, int32_t *out);
int moe_debug_silu_mul(int dtype, const void *gate_up, void *act, int64_t M, int I, cudaStream_t stream);

// paro_moe_grouped.cu
size_t moe_grouped_workspace_bytes(const paro_moe_desc *d, int64_t T, int32_t k);
int moe_grouped_forward(const paro_moe_desc *d, const void *x, const int32_t *ids, const float *wts, int64_t T, int32_t k, void *h, void *y,
                        void *workspace, size_t workspace_bytes, cudaStream_t stream);
int moe_grouped_debug_plan(const paro_moe_desc *d, int64_t T, int32_t k, int32_t *out);

// paro_moe_route.cu
int moe_route_forward(const void *x, const void *w, int dtype, int64_t T, int hidden, int E, int k, int renormalize, int32_t *ids, float *wts,
                      float *logits, cudaStream_t stream);
int moe_route_debug_plan(int64_t T, int hidden, int E, int k, int sms, int32_t *out);

}  // namespace paro
