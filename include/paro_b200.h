/*
 * paro_b200.h -- C ABI of libparo_b200.so: the sm_90a (H100) implementation of ParoQuant's
 * hot path (scaled pairwise rotation of the activations + AWQ INT4 group dequant + GEMV/GEMM).
 *
 * Plain pointers and sizes only; no torch / ATen types.  Every pointer named "device" must be
 * device memory of the CUDA device that is current on the calling thread; `stream` is a
 * cudaStream_t.  No entry point allocates, synchronises the host, or keeps mutable global
 * state, so all of them are safe under CUDA-graph capture and re-entrant across streams (a
 * `workspace` must not be shared by launches that may run concurrently).
 *
 * Each entry point replaces one piece of the reference's operator surface (paths relative to
 * the z-lab/paroquant tree):
 *
 *   paro_rotate            torch.ops.rotation.rotate
 *                            paroquant/kernels/cuda/rotation.cu:10-43   (kernel)
 *                            paroquant/kernels/cuda/rotation.cu:62-95   (launcher, dtype casts)
 *                            paroquant/kernels/cuda/rotation.cu:111-135 (dispatch + schema)
 *   paro_packed_bytes /    the AWQ -> kernel-layout repack the reference does through Marlin in
 *   paro_prepack             ParoQuantLinearMethod.process_weights_after_loading
 *                            paroquant/inference/backends/vllm/plugin.py:208-279
 *   paro_workspace_bytes   Marlin's per-layer workspace (plugin.py:249,272)
 *   paro_linear_forward    ParoQuantLinearMethod.apply   plugin.py:281-311  (rotate + Marlin,
 *                            per partition, cat, bias) and RotateQuantizedLinear.forward
 *                            paroquant/inference/backends/transformers/modules.py:57-71
 *   paro_last_error        TORCH_CHECK messages of rotation.cu:66,92,108,114,123
 *   paro_moe_forward       RotateSwitchGLU  paroquant/inference/backends/mlx/modules.py:159-212 on the
 *   paro_moe_grouped_forward expert format of paroquant/cli/convert.py:281-406 (decode batches / any batch)
 *
 * Return value of every int function: 0 on success, a PARO_E* code otherwise; the message is
 * available from paro_last_error() on the same thread.
 */
#ifndef PARO_B200_H_
#define PARO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PARO_ABI_VERSION 5
#define PARO_MAX_PARTS 8

/* element types (activations, rotation parameters, scales) */
#define PARO_F32 0
#define PARO_F16 1
#define PARO_BF16 2

/* error codes */
#define PARO_OK 0
#define PARO_EINVAL 1      /* bad shape / dtype / null pointer / alignment */
#define PARO_EUNSUPPORTED 2 /* valid request this build has no kernel for   */
#define PARO_ECUDA 3       /* CUDA runtime error (message carries cudaGetErrorString) */
#define PARO_EWORKSPACE 4  /* workspace too small */

typedef void *paro_stream_t; /* cudaStream_t */

/* Geometry of one (possibly merged) quantised linear as this rank sees it.
 * Mirrors what ParoQuantLinearMethod.create_weights receives (plugin.py:173-206):
 * in_features = input_size_per_partition, part_sizes = output_partition_sizes.        */
typedef struct paro_linear_shape {
  int32_t in_features;                 /* K, multiple of 128                           */
  int32_t out_features;                /* N = sum(part_sizes)                          */
  int32_t group_size;                  /* quantisation == rotation group; 64 or 128    */
  int32_t krot;                        /* rotations per group (1..16); 8 in checkpoints */
  int32_t n_parts;                     /* 1, or 3 for QKV / 2 for gate_up              */
  int32_t part_sizes[PARO_MAX_PARTS];  /* each a multiple of 16                        */
  int32_t dtype;                       /* activation / output dtype: PARO_F16 | PARO_BF16 */
} paro_linear_shape;

int paro_abi_version(void);
const char *paro_last_error(void);

/* out[m, g*G + c] = (prod_r Givens_r)(x[m, g*G + :] * scales) -- torch.ops.rotation.rotate.
 *   x, out      device [M, K] of `dtype` (F32 | F16 | BF16), contiguous; out may alias x
 *   idx_ij      device [krot, K] int16, local pair indices (i at 2t, j at 2t+1)
 *   theta       device [krot, K/2] of theta_dtype; cast to `dtype` before use exactly like
 *               rotation.cu:75 does (`theta.to(x.dtype)`), but inside the kernel
 *   scales      device [K] of scales_dtype or NULL (rotation.cu:76-78)
 *   group_size  64 or 128 (rotation.cu:117-123); krot 1..16
 * Rounding points are those of rotation.cuh:91-173 (fp16/bf16) and :16-75 (fp32).       */
int paro_rotate(const void *x, void *out, const int16_t *idx_ij, const void *theta,
                int32_t theta_dtype, const void *scales, int32_t scales_dtype, int64_t M,
                int32_t K, int32_t krot, int32_t group_size, int32_t dtype, paro_stream_t stream);

/* Backward of paro_rotate in ONE launch -- replaces RotateTensorFunc.backward's Python walk over the rotations
 * (kernels/cuda/autograd.py:20-61: per rotation two rotate launches, five gathers and a reduction).
 *   y           device [M, K] of `dtype`: the forward OUTPUT;  grad_out [M, K]: dL/dy
 *   x           device [M, K]: the forward input, read only when grad_scale != NULL
 *   grad_x      device [M, K] of `dtype` (written);  must not alias y / grad_out
 *   grad_theta  device [krot, K/2] fp32, ACCUMULATED into (zero it first)
 *   grad_scale  device [K] fp32, accumulated into, or NULL (then scales may be NULL too)
 * t and g are rounded to `dtype` after every rotation, where the reference's per-rotation
 * launches store them; the sums over rows run in fp32 (atomics: order-dependent last bits).
 * theta_formula  PARO_THETA_GRADIENT: grad_theta = sum_rows (g_i t_j - g_j t_i) per pair, the gradient;
 *                PARO_THETA_REFERENCE_EXPRESSION: the value the reference's expression takes
 *                (autograd.py:50-52, applied after g was un-rotated too, autograd.py:38):
 *                cos * gradient - sin * sum_rows(g . t) -- see paroquant_b200/kernels/cuda/autograd.py.
 * grad_x and grad_scale equal the reference's either way.                                            */
#define PARO_THETA_GRADIENT 0
#define PARO_THETA_REFERENCE_EXPRESSION 1
int paro_rotate_backward(const void *y, const void *grad_out, const void *x, const int16_t *idx_ij,
                         const void *theta, int32_t theta_dtype, const void *scales, int32_t scales_dtype,
                         void *grad_x, float *grad_theta, float *grad_scale, int64_t M, int32_t K,
                         int32_t krot, int32_t group_size, int32_t dtype, int32_t theta_formula,
                         paro_stream_t stream);

/* Test hook (host only, no device work): the launch plan of paro_rotate_backward on a device with `sms` SMs, the function the
 * launch itself uses.  out[0] = dynamic shared-memory bytes per CTA, out[1] = CTAs per SM it plans for, out[2] = splits (warps
 * per group; warp `split` walks row blocks split, split + splits, ...), out[3] = row blocks of 4 rows, out[4] / out[5] = the
 * most / fewest row blocks one warp walks, out[6] = grid CTAs.  M >= 1; the other arguments as paro_rotate_backward takes them. */
int paro_debug_rotate_backward_plan(int64_t M, int32_t K, int32_t krot, int32_t group_size, int32_t dtype,
                                    int32_t theta_formula, int32_t sms, int64_t *out);

/* Size in bytes of the kernel-layout buffer paro_prepack fills (0 on invalid shape). */
size_t paro_packed_bytes(const paro_linear_shape *shape);

/* One-time repack of checkpoint-format buffers into the streaming layout of the fused kernels.
 *   qweight  device [K, N/8] int32, AWQ nibble order (convert.py:19,149-155)
 *   qzeros   device [K/G, N/8] int32
 *   scales   device [K/G, N] of scales_dtype (fp16 on disk; vLLM holds them in the model dtype)
 *   pairs    device [n_parts, krot, K] int16
 *   theta    device [n_parts, krot, K/2] of theta_dtype
 *   channel_scales device [n_parts, K] of cs_dtype
 *   packed   device, paro_packed_bytes(shape) bytes, 128-byte aligned
 * Values are preserved exactly: the kernels reproduce T((q - z) * T(s)) and the reference
 * rotation bit for bit; only the layout changes.                                         */
int paro_prepack(const paro_linear_shape *shape, const int32_t *qweight, const int32_t *qzeros,
                 const void *scales, int32_t scales_dtype, const int16_t *pairs,
                 const void *theta, int32_t theta_dtype, const void *channel_scales,
                 int32_t cs_dtype, void *packed, paro_stream_t stream);

/* Bytes of scratch paro_linear_forward needs for up to max_m rows.  Head: the small-M kernel's block counters
 * (they must be ZERO when the buffer is first used; every launch leaves them zeroed); behind them pure scratch: the
 * fp32 partial slots of the M <= 16 kernel or the rotated activations of the M > 16 path (n_parts x M x K elements).  */
size_t paro_workspace_bytes(const paro_linear_shape *shape, int64_t max_m);

/* y[M, N] = rotate_p(x) . dequant(W)[:, part p] for every partition p (+ bias) in ONE call.
 *   packed     device buffer from paro_prepack
 *   x          device [M, K] of shape->dtype, contiguous
 *   bias       device [N] of shape->dtype or NULL
 *   y          device [M, N] of shape->dtype
 *   workspace  device, >= paro_workspace_bytes(shape, M), 256-byte aligned
 * M <= 16 runs the fused rotate+dequant+GEMV kernel (HBM-bound); larger M the
 * rotate + wgmma GEMM path.                                                            */
int paro_linear_forward(const paro_linear_shape *shape, const void *packed, const void *x,
                        int64_t M, const void *bias, void *y, void *workspace,
                        size_t workspace_bytes, paro_stream_t stream);

/* ---- chains: several linears of one decode step (M <= 16) in ONE launch, element-wise neighbours folded in ----------
 * The reference runs every quantised linear as its own rotate + GEMM kernels (plugin.py:281-311) and leaves what sits
 * between them to vLLM: fused_add_rms_norm before qkv / gate_up, silu_and_mul before down, the residual add after o /
 * down (call sites of ParoQuantLinearMethod.apply).  A chain runs up to PARO_CHAIN_MAX_STEPS such linears back to back
 * inside one persistent kernel: the weight stream of step i + 1 is prefetched while step i drains, and the neighbours
 * become the x op / epilogue of the adjacent step.                                                                   */
#define PARO_CHAIN_MAX_STEPS 6
#define PARO_XOP_NONE 0      /* x as given                                                                          */
#define PARO_XOP_SILU_MUL 1  /* x[m, k] = T(silu(g[m, k])) * u[m, k]; input is [M, 2K] = [gate | up]  (silu_and_mul) */
#define PARO_XOP_RMSNORM 2   /* x = T(T(h * rstd) * w), rstd from the previous step's ADD_RESIDUAL statistics        */
#define PARO_EPI_STORE 0         /* y = T(acc) (+ bias)                                                             */
#define PARO_EPI_ADD_RESIDUAL 1  /* h = T(y + residual_in) -> residual_out (fused_add_rms_norm's first half)        */

/* Tensor parallelism inside a step (row-sharded K: o_proj / down_proj, reference sharding plugin.py:33-50): every rank's
 * block sums are written into every rank's `peer_slots` buffer over NVLink and added in rank order by the kernel itself --
 * the all-reduce vLLM issues after ParoQuantLinearMethod.apply (RowParallelLinear.forward) happens inside the launch.
 * peer_slots[r] = device address, valid on THIS GPU, of rank r's buffer of paro_tp_slot_bytes() bytes (peer-mapped memory:
 * CUDA IPC / symmetric memory), zero-filled once.  All ranks must launch the same chains in the same order.            */
#define PARO_TP_MAX_RANKS 8
typedef struct paro_tp_info {
  int32_t world, rank;
  void *peer_slots[PARO_TP_MAX_RANKS];
} paro_tp_info;

typedef struct paro_chain_step {
  const paro_linear_shape *shape;
  const void *packed;        /* device, from paro_prepack                                                          */
  const void *bias;          /* device [N] or NULL                                                                 */
  const void *x;             /* device input, ready at launch; NULL = the previous step's output (y, or
                              * residual_out after an ADD_RESIDUAL epilogue)                                         */
  void *y;                   /* device [M, N]; may be NULL with PARO_EPI_ADD_RESIDUAL                               */
  int32_t x_op;              /* PARO_XOP_*                                                                          */
  int32_t epilogue;          /* PARO_EPI_*                                                                          */
  const void *residual_in;   /* ADD_RESIDUAL: device [M, N]                                                         */
  void *residual_out;        /* ADD_RESIDUAL: device [M, N], must not alias residual_in                             */
  const void *norm_weight;   /* RMSNORM: device [K] of shape->dtype                                                 */
  float eps;                 /* RMSNORM                                                                             */
  const paro_tp_info *tp;    /* NULL, or: this step's K is sharded over tp->world ranks, sum the partial outputs      */
} paro_chain_step;

/* Bytes of the per-rank peer_slots buffer of one tensor-parallel step (0 on an invalid shape).                        */
size_t paro_tp_slot_bytes(const paro_linear_shape *shape, int64_t M, int32_t world);

/* Workspace bytes for paro_chain_forward (0 on an invalid chain).  The workspace must be zero-filled once when it is
 * allocated; every launch leaves its counters zeroed again.                                                        */
size_t paro_chain_workspace_bytes(const paro_chain_step *steps, int32_t n_steps, int64_t M);

/* Run the chain for M <= 16 rows.  One launch; CUDA-graph safe; no allocation, no host synchronisation.             */
int paro_chain_forward(const paro_chain_step *steps, int32_t n_steps, int64_t M, void *workspace,
                       size_t workspace_bytes, paro_stream_t stream);

/* ---- prefill chains: the same step descriptors for any M >= 1 (prefill chunks, more than 16 sequences in flight) --------
 * Every step is the M > 16 path of paro_linear_forward -- the rotation pre-pass, then the INT4 wgmma GEMM -- with the step's
 * x op in the pre-pass and its epilogue in the GEMM (paroquant_b200/csrc/paro_gemm.cu).  Each step computes what the decode
 * chain computes: SILU_MUL is paro_debug_silu_mul's operand bit for bit; RMSNORM is T(T(h * rstd) * w) with rstd =
 * rsqrtf(sum(h^2) / K + eps) of the previous step's residual_out; STORE gives y = T(acc), then + bias in T; ADD_RESIDUAL
 * stores t = T(acc) (+ bias in T) to y where y is given and h = T(t + residual_in) to residual_out.  Output row m depends only
 * on the inputs' row m, in a fixed summation order (the RMSNorm statistics too): results are bit-reproducible and do not
 * depend on the other rows of the batch.  Checks and messages are the decode chain's; steps with tp->world > 1 give
 * PARO_EUNSUPPORTED.  2 x n_steps launches (paro_last_launch_count()); CUDA-graph safe; no allocation, no host
 * synchronisation.
 * Workspace bytes for paro_prefill_chain_forward (0 on an invalid chain): pure scratch, nothing persists between calls --
 * the rotated operand of the largest step, fp32 row statistics of every ADD_RESIDUAL step an RMSNORM step consumes, and the
 * outputs of consumed STORE steps without y.                                                                             */
size_t paro_prefill_chain_workspace_bytes(const paro_chain_step *steps, int32_t n_steps, int64_t M);

/* Run the chain for M >= 1 rows; workspace 256-byte aligned, below paro_prefill_chain_workspace_bytes gives
 * PARO_EWORKSPACE.                                                                                                      */
int paro_prefill_chain_forward(const paro_chain_step *steps, int32_t n_steps, int64_t M, void *workspace,
                               size_t workspace_bytes, paro_stream_t stream);

/* ---- MoE expert block for decode batches: the routed experts of one block in TWO launches, routing read on the device ----
 * Replaces the reference's RotateSwitchGLU (paroquant/inference/backends/mlx/modules.py:159-212) on the expert format of
 * paroquant/cli/convert.py:281-406: every expert is a merged gate|up linear and a down linear, and all experts share ONE
 * gate_up rotation and ONE down rotation.  For token t and slot s with e = topk_ids[t, s] in [0, n_experts):
 *   h[t, s]  = T(rotate_gu(x[t]) . W_gu[e])                              (2I outputs: gate | up)
 *   y_s      = T(rotate_d(T(T(silu(gate)) * up)) . W_d[e])
 *   y[t]     = T(sum of fp32(y_s) * w_s, from 0, in ascending (expert id, slot) order, each product rounded before its add)
 * A slot whose id lies outside [0, n_experts) contributes nothing (expert parallelism marks non-local experts with -1);
 * duplicate ids in one token each contribute.  Two PDL-chained launches, no host synchronisation, no allocation; one
 * launch plan serves every routing, so a captured CUDA graph stays valid while the ids / weights in its buffers change.  */
typedef struct paro_moe_desc {
  const paro_linear_shape *gate_up;  /* every expert's merged gate|up: in_features = hidden, parts {I, I}               */
  const paro_linear_shape *down;     /* every expert's down: in_features = I, parts {hidden}                            */
  int32_t n_experts;
  const void *gate_up_packed;        /* device; expert e's paro_prepack buffer at + e * gate_up_stride                  */
  size_t gate_up_stride;             /* >= paro_packed_bytes(gate_up), multiple of 256                                  */
  const void *down_packed;
  size_t down_stride;
} paro_moe_desc;

/* Workspace bytes for paro_moe_forward (0 on an invalid descriptor or batch).                                          */
size_t paro_moe_workspace_bytes(const paro_moe_desc *d, int64_t T, int32_t top_k);

/* Run the expert block for T tokens with top_k slots each.
 *   x             device [T, hidden] of the shapes' dtype
 *   topk_ids      device [T, top_k] int32;  topk_weights device [T, top_k] fp32
 *   h             device [T, top_k, 2I]: the gate|up outputs (rows of dropped slots are left unspecified)
 *   y             device [T, hidden]
 * 1 <= T <= 16, 1 <= top_k <= 16 and T * top_k <= 128 (the routing table is built by one thread per entry in shared
 * memory); otherwise PARO_EUNSUPPORTED.  paro_last_launch_count() reports 2.                                          */
int paro_moe_forward(const paro_moe_desc *d, const void *x, const int32_t *topk_ids, const float *topk_weights,
                     int64_t T, int32_t top_k, void *h, void *y, void *workspace, size_t workspace_bytes,
                     paro_stream_t stream);

/* Test hook (host only): the two launch plans of paro_moe_forward on a device with `sms` SMs and a walk of their work
 * lists.  out[0..7] gate_up, out[8..15] down: cluster size, K slices per expert, grid, output blocks, groups, max groups
 * per work item, ring stages, shared-memory bytes; out[16] = U_max = min(n_experts, T * top_k); out[17] = the number of
 * coverage violations over U = 1..U_max (a (expert slot, group) round of a block owned other than exactly once, or rank 0
 * reading a receive slot no rank wrote in that wave).                                                                  */
int paro_debug_moe_plan(const paro_moe_desc *d, int64_t T, int32_t top_k, int32_t sms, int32_t *out);

/* ---- MoE expert block for any batch: the routed experts as grouped INT4 wgmma GEMMs, routing read on the device ----------
 * Same descriptor, semantics, alignments and checks as paro_moe_forward, for batches the decode kernel does not take (prefill,
 * or more than 16 sequences in flight).  Six launches (paroquant_b200/csrc/paro_moe_grouped.cu): the routing table (entries
 * sorted by expert, each expert's run padded to whole tiles of NT rows), the gate_up pre-pass (x gathered through the table,
 * rotated once per entry), the grouped gate_up GEMM (scattered to h), the down pre-pass (SiLU * up of h, rotated), the grouped
 * down GEMM (into the workspace) and the per-token combine.  No host synchronisation, no allocation; the plan depends on
 * (T, top_k, n_experts) only, so a captured CUDA graph stays valid while the ids / weights in its buffers change.  Every
 * h[t, s] and y_s row is computed independently of the tiling: permuting tokens or slots permutes h and y bit for bit.
 * paro_last_launch_count() reports 6.                                                                                     */
#define PARO_MOE_GROUPED_MAX_ENTRIES 65536   /* T * top_k                                                                   */
#define PARO_MOE_GROUPED_MAX_EXPERTS 1024

/* Workspace bytes for paro_moe_grouped_forward (0 on an invalid descriptor or batch): the routing table, the rotated operand
 * of both GEMMs (tiles_max x NT rows of max(hidden, I) elements) and the y_s rows (T x top_k x hidden elements).           */
size_t paro_moe_grouped_workspace_bytes(const paro_moe_desc *d, int64_t T, int32_t top_k);

/* Run the expert block for T tokens with top_k slots each; arguments as paro_moe_forward, workspace 256-byte aligned.
 * 1 <= top_k <= 16, T >= 1, T * top_k <= PARO_MOE_GROUPED_MAX_ENTRIES and n_experts <= PARO_MOE_GROUPED_MAX_EXPERTS;
 * otherwise PARO_EUNSUPPORTED.  A workspace below paro_moe_grouped_workspace_bytes gives PARO_EWORKSPACE.              */
int paro_moe_grouped_forward(const paro_moe_desc *d, const void *x, const int32_t *topk_ids, const float *topk_weights,
                             int64_t T, int32_t top_k, void *h, void *y, void *workspace, size_t workspace_bytes,
                             paro_stream_t stream);

/* Test hook (host only): the plan of paro_moe_grouped_forward.  out[0] = NT (rows per tile: 32, 64 or 128), out[1] = tiles_max
 * = floor(T * top_k / NT) + min(n_experts, T * top_k), out[2..7] = grid of each launch (route, gate_up pre-pass, gate_up GEMM,
 * down pre-pass, down GEMM, combine), out[8..11] = workspace bytes / 256 of the routing table, the operand, the y_s rows and
 * in total.  The plan does not depend on the SM count; `sms` must be >= 1.                                                */
int paro_debug_moe_grouped_plan(const paro_moe_desc *d, int64_t T, int32_t top_k, int32_t sms, int32_t *out);

/* ---- MoE router: logits, softmax and top-k of a block in ONE launch, written where the two expert-block entry points read ----
 * For x [T, hidden] and the router weight router_w [n_experts, hidden] (row-major, as a checkpoint stores mlp.gate.weight; no
 * prepack), both of dtype D (PARO_F16 | PARO_BF16):
 *   logit[t, e]        = D(sum_h x[t, h] * w[e, h])          fp32 accumulation, one rounding to D
 *   p[t, :]            = softmax(fp32(logit[t, :]))          fp32, max subtracted first
 *   slots              = the top_k experts by descending logit; equal logits -> lower expert id first; slot 0 is the largest
 *   topk_weights[t, s] = p[t, id_s]                          (renormalize = 0)
 *                      = p[t, id_s] / sum_s' p[t, id_s']     (renormalize = 1, the sum taken in slot order)
 *   topk_ids[t, s]     = id_s
 * (softmax -> top-k -> optional renormalise, as Qwen3-MoE's norm_topk_prob and Mixtral route).  logits_or_null, when given,
 * receives the fp32 values of the D-rounded logits, [T, n_experts].  Row t of every output depends on row t of x and on router_w
 * only: hidden is cut into K slices fixed by hidden alone and the slice sums are added in slice order, whatever T, the row's
 * position in the batch and the launch plan -- a token routes bit-identically in a 1-token step and inside a prefill chunk.
 * hidden a multiple of 128, 1 <= n_experts <= 256, 1 <= top_k <= min(n_experts, 16); otherwise PARO_EUNSUPPORTED.  x and
 * router_w 16-byte, the outputs 4-byte aligned.  T = 0 succeeds without a launch.  One launch (paro_last_launch_count() reports
 * 1), no workspace, no allocation, no host synchronisation; CUDA-graph safe.  The kernel releases its programmatic dependents
 * at once: paro_moe_forward's kernels, launched next in the stream, start their prologue under it and wait for its completion
 * before they read the routing.                                                                                              */
int paro_moe_route(const void *x, const void *router_w, int32_t dtype, int64_t T, int32_t hidden, int32_t n_experts,
                   int32_t top_k, int32_t renormalize, int32_t *topk_ids, float *topk_weights, float *logits_or_null,
                   paro_stream_t stream);

/* Test hook (host only): the plan of paro_moe_route on a device with `sms` SMs.  out[0] = NT (tokens per tile: 8, 16 or 32),
 * out[1] = cluster size c (1, 2, 4 or 8 CTAs per token tile), out[2] = K slices (a function of hidden alone), out[3] = grid,
 * out[4] = shared-memory bytes, out[5] = the number of coverage violations from a walk of the plan (a (token tile, K slice)
 * owned other than exactly once), out[6] = token tiles, out[7] = threads per CTA.  T >= 1.                                  */
int paro_debug_moe_route_plan(int64_t T, int32_t hidden, int32_t n_experts, int32_t top_k, int32_t sms, int32_t *out);

/* Debug / test aid: dequantise the prepacked weights back to a dense [K, N] matrix of
 * shape->dtype (the exact operand the GEMM consumes).                                    */
int paro_unpack_dense(const paro_linear_shape *shape, const void *packed, void *W_out,
                      paro_stream_t stream);

/* Debug / test aid: act[m, i] = T(T(silu(gate[m, i])) * up[m, i]) for device gate_up [M, 2I] (gate | up) and act [M, I]
 * of dtype (PARO_F16 | PARO_BF16), both 4-byte aligned, I even.  The library's own SiLU * up, bit-identical to the
 * operand paro_moe_forward's down launch and the chains' PARO_XOP_SILU_MUL step rotate (its exp is the fast one, which
 * an fp32 or fp64 exp does not reproduce bit for bit).                                                                */
int paro_debug_silu_mul(int32_t dtype, const void *gate_up, void *act, int64_t M, int32_t I, paro_stream_t stream);

/* Number of kernels the last successful paro_linear_forward / paro_rotate call on this
 * thread launched (bench.py's gpu_launches accounting).                                  */
int paro_last_launch_count(void);

/* Test hook (host only, no device work): the launch plan of the M <= 16 kernel for a device with `sms` SMs that keeps
 * resident_clusters[log2 c] clusters of c = 1, 2, 4, 8 CTAs resident.  out[0..10] = cluster size, block ranges, grid,
 * max blocks per CTA, max groups per CTA, ring stages, rotating warps, shared-memory bytes, B-operand / receive /
 * barrier offsets; out[11..19] = first block range of every partition (+ end).                                    */
int paro_debug_decode_plan(const paro_linear_shape *shape, int64_t M, int32_t sets, int32_t sms,
                           const int32_t *resident_clusters, int32_t *out);

/* Test hook (host only): the plan of one step of the small-M kernel on `ctas` CTAs.  out[0..4] = K slices, members per
 * slice, max contributor slots per block, max groups per CTA, max rounds per CTA; out[5..13] = first member of every
 * partition's team (+ end).                                                                                          */
int paro_debug_stream_plan(const paro_linear_shape *shape, int64_t M, int32_t sets, int32_t ctas, int32_t *out);

/* Test hook (host only): the tile of the M > 16 GEMM on a device with `sms` SMs.  out[0] = tokens per output tile (32, 64
 * or 128), out[1] = token blocks (tiles along M; the last one is partial unless NT divides M).                       */
int paro_debug_gemm_plan(const paro_linear_shape *shape, int64_t M, int32_t sms, int32_t *out);

/* Developer aid: with PARO_DECODE_TRACE=1 the small-M kernel records, per CTA and step, 8 timestamps (SM cycles since
 * kernel entry).  Copies the first max_ctas x PARO_CHAIN_MAX_STEPS x 8 values of the last launch to host_out.        */
int paro_debug_stream_trace(unsigned long long *host_out, int32_t max_ctas);

/* Developer aid: with PARO_DECODE_TRACE=1 in the environment the small-M kernel records, per CTA,
 * 12 uint64 values (phase timestamps in SM cycles relative to kernel entry, %globaltimer at entry
 * and exit).  Copies the first max_ctas x 12 values of the last launch to host_out (synchronous). */
int paro_debug_trace(unsigned long long *host_out, int32_t max_ctas);

#ifdef __cplusplus
}
#endif
#endif /* PARO_B200_H_ */
