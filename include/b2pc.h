/*
 * b2pc.h -- C ABI of libb2pc.so, the H100 (sm_90a) point-cloud backbone operator library.
 *
 * This is the drop-in boundary for the two third-party operator packages Pointcept's
 * PT-v3m1 / SpUNet-v1m1 hot path calls (the reference itself has no C ABI: its in-repo
 * extensions bind at::Tensor through pybind11, e.g. libs/pointops/src/pointops_api.cpp:15-32,
 * and the hot-path arithmetic lives in the spconv / flash-attn wheels).  Each entry point
 * names the reference call site it serves.
 *
 * Conventions
 *   - every function returns 0 on success or a negative b2pc_status; b2pc_last_error()
 *     returns a thread-local message for the last failure on the calling thread;
 *   - all data pointers are DEVICE pointers unless the parameter name ends in _host;
 *   - functions never allocate, free or synchronise: the caller owns every buffer, passes
 *     scratch memory obtained from the matching *_workspace_bytes() query, and passes the
 *     CUDA stream to launch on (cudaStream_t == b2pc_stream_t);
 *   - re-entrant and thread-safe (forward on the main thread, backward on autograd's
 *     device thread; one process per GPU as in pointcept/engines/launch.py:73);
 *   - dtype enum: 0 = fp32, 1 = fp16, 2 = bf16 (features/weights; accumulation is fp32).
 */
#ifndef B2PC_H_
#define B2PC_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* b2pc_stream_t;

typedef enum {
  B2PC_OK = 0,
  B2PC_ERR_INVALID_ARG = -1,
  B2PC_ERR_WORKSPACE = -2,
  B2PC_ERR_CUDA = -3,
  B2PC_ERR_UNSUPPORTED = -4
} b2pc_status;

enum { B2PC_F32 = 0, B2PC_F16 = 1, B2PC_BF16 = 2 };
/* serialization orders, pointcept/models/utils/serialization/default.py:10-18 */
enum { B2PC_ORDER_Z = 0, B2PC_ORDER_Z_TRANS = 1, B2PC_ORDER_HILBERT = 2, B2PC_ORDER_HILBERT_TRANS = 3 };

int b2pc_version(void);
const char* b2pc_last_error(void);
/* number of CUDA kernels this library has launched in this process (bench.py's gpu_launches) */
long long b2pc_launch_count(void);

/* ---------------------------------------------------------------------------------------------
 * Serialization: replaces encode() (serialization/default.py:9-24, z_order.py:66-101,
 * hilbert.py:91-192) and the argsort / inverse scatter of Point.serialization
 * (models/utils/structure.py:85-100).
 * ------------------------------------------------------------------------------------------- */

/* code[o, i] = (batch[i] << 3*depth) | curve_{orders_host[o]}(grid_coord[i]);  all requested
 * orders in one pass over the coordinates.  grid_coord [N,3] int32, batch [N] int64 or NULL,
 * code [n_orders, N] int64.  1 <= depth <= 16, n_orders <= 8. */
int b2pc_serialize_encode(const int32_t* grid_coord, const int64_t* batch, int64_t n, int depth,
                          const int* orders_host, int n_orders, int64_t* code, b2pc_stream_t stream);

size_t b2pc_serialize_sort_workspace_bytes(int64_t n, int n_orders);
/* Stable LSD radix sort of every row of code[n_orders, N] on its low key_bits bits
 * (key_bits = 3*depth + bits(batch_size-1); <= 63).  order[o] = argsort(code[o]) (int64, as
 * torch.argsort returns), inverse[o][order[o][i]] = i.  Only the significant bits are sorted. */
int b2pc_serialize_sort(const int64_t* code, int64_t n, int n_orders, int key_bits, int64_t* order,
                        int64_t* inverse, void* workspace, size_t workspace_bytes,
                        b2pc_stream_t stream);

/* Patch padding tables: replaces SerializedAttention.get_padding_and_inverse
 * (point_transformer_v3/point_transformer_v3m1_base.py:114-170) without its per-scene host loop.
 * offset [B] int64 (device, cumulative scene sizes).  The caller knows the scene sizes on the
 * host and passes t_pad = sum of padded sizes and n_seq = number of patches.
 * pad [t_pad] int64, unpad [n] int64, cu_seqlens [n_seq+1] int32. */
int b2pc_patch_padding(const int64_t* offset, int batch_size, int patch_size, int64_t n, int64_t t_pad,
                       int n_seq, int64_t* pad, int64_t* unpad, int32_t* cu_seqlens,
                       b2pc_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Patch attention: replaces flash_attn.flash_attn_varlen_qkvpacked_func as called at
 * point_transformer_v3m1_base.py:208-214 (non-causal, no dropout, no mask).
 * qkv [T,3,H,D] contiguous (fp16 or bf16), cu_seqlens [n_seq+1] int32, out [T,H,D] (same dtype),
 * lse [H,T] fp32 (natural-log sum-exp of scale*QK^T, flash-attn's softmax_lse layout).
 * impl: 0 = auto (tensor-core kernel when the shape is supported), 1 = SIMT reference kernel,
 *       2 = tensor-core kernel (error if unsupported).
 * ------------------------------------------------------------------------------------------- */
int b2pc_patch_attn_fwd(const void* qkv, int dtype, const int32_t* cu_seqlens, int n_seq, int max_seqlen,
                        int64_t t, int heads, int head_dim, float scale, void* out, float* lse,
                        int impl, b2pc_stream_t stream);

size_t b2pc_patch_attn_bwd_workspace_bytes(int64_t t, int heads, int head_dim);
/* dqkv [T,3,H,D] (same dtype) from dout [T,H,D], the forward's qkv / out / lse. */
int b2pc_patch_attn_bwd(const void* dout, const void* qkv, const void* out, const float* lse, int dtype,
                        const int32_t* cu_seqlens, int n_seq, int max_seqlen, int64_t t, int heads,
                        int head_dim, float scale, void* dqkv, void* workspace, size_t workspace_bytes,
                        int impl, b2pc_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Sparse convolution rulebooks: replaces the indice-pair generation inside
 * spconv.pytorch.SubMConv3d / SparseConv3d (call sites: point_transformer_v3m1_base.py:278-284,
 * 499-506; sparse_unet/spconv_unet_v1m1_base.py:43-68,114-121,137-144,173-179,222-224).
 * indices [N,4] int32 rows (b, x, y, z) as built at models/utils/structure.py:139-146.
 * Rulebook form: pair[KV, N_out] int32, entry = input row feeding output row j through kernel
 * offset k = (i0*K1+i1)*K2+i2, or -1.
 * ------------------------------------------------------------------------------------------- */
size_t b2pc_rulebook_workspace_bytes(int64_t n, int reach);   /* submanifold: reach = 1 */
/* strided: sized for n * reach distinct outputs, reach = prod_axis ceil(k / (s / gcd(s, d))) (1 for k = 2, s = 2) */
size_t b2pc_rulebook_strided_workspace_bytes(int64_t n, const int* ksize_host, const int* stride_host, const int* dilation_host);
/* Submanifold: output set == input set (same rows); padding is implied (K//2 * dilation). */
int b2pc_rulebook_subm(const int32_t* indices, int64_t n, const int* spatial_shape_host,
                       const int* ksize_host, const int* dilation_host, int32_t* pair,
                       void* workspace, size_t workspace_bytes, b2pc_stream_t stream);
/* Strided (SparseConv3d): out coordinate o is active iff some input i and offset k satisfy
 * i = o*stride - padding + k*dilation.  Output rows are the distinct out coordinates in
 * ascending (b,x,y,z) order.  Two stages because M is data dependent: _begin writes num_out[0] = number of distinct
 * outputs and num_out[1] = largest batch index (device int64[2]); the caller reads both (one host sync, as spconv does),
 * passes M and batch_count = num_out[1] + 1 (bounds the sort key width; 0 = unknown) to _finish,
 * allocates out_indices [M,4], pair_fwd [KV,M], pair_bwd [KV,N] and calls _finish with the SAME
 * workspace (its contents carry over). */
int b2pc_rulebook_strided_begin(const int32_t* indices, int64_t n, const int* spatial_shape_host,
                                const int* ksize_host, const int* stride_host, const int* padding_host,
                                const int* dilation_host, int64_t* num_out, void* workspace,
                                size_t workspace_bytes, b2pc_stream_t stream);
int b2pc_rulebook_strided_finish(const int32_t* indices, int64_t n, const int* spatial_shape_host,
                                 const int* ksize_host, const int* stride_host, const int* padding_host,
                                 const int* dilation_host, int64_t num_out_host, int batch_count_host, int32_t* out_indices,
                                 int32_t* pair_fwd, int32_t* pair_bwd, void* workspace,
                                 size_t workspace_bytes, b2pc_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Sparse convolution arithmetic (gather - GEMM - accumulate, output stationary, no atomics):
 *   out[j, :] = bias + sum_k  in[pair[k', j], :] @ W_k          k' = flip ? KV-1-k : k
 * Forward:        W_k = weight[:, k, :]^T   (weight [Cout, KV, Cin], the spconv parameter layout)
 * Backward data:  same routine on dout with transpose_w = 1 (W_k = weight[:, k, :], [Cout]->[Cin]);
 *                 SubM passes the forward table with flip = 1 (the table is its own inverse under
 *                 k -> KV-1-k), strided / inverse convs pass the opposite-direction table.
 * n_in rows of feat, n_out rows of out / columns of pair.  impl as for attention.
 * ------------------------------------------------------------------------------------------- */
size_t b2pc_spconv_gather_gemm_workspace_bytes(int64_t n_out, int c_in, int c_out, int kv);
int b2pc_spconv_gather_gemm(const void* feat, const void* weight, const void* bias, const int32_t* pair,
                            int64_t pair_stride, int64_t n_in, int64_t n_out, int c_in, int c_out, int kv,
                            int transpose_w, int flip, int dtype, void* out, void* workspace,
                            size_t workspace_bytes, int impl, b2pc_stream_t stream);

size_t b2pc_spconv_bwd_weight_workspace_bytes(int64_t n_out, int c_in, int c_out, int kv);
/* dweight[co, k, ci] = sum_j  dout[j, co] * feat_in[pair[k, j], ci]   (fp32 result, deterministic). */
int b2pc_spconv_bwd_weight(const void* feat_in, const void* dout, const int32_t* pair, int64_t pair_stride,
                           int64_t n_in, int64_t n_out, int c_in, int c_out, int kv, int dtype,
                           float* dweight, void* workspace, size_t workspace_bytes, int impl,
                           b2pc_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Serialized pooling (SURVEY.md 8(f).1): replaces proj(feat)[indices] + torch_scatter.segment_csr(max)
 * of SerializedPooling.forward (point_transformer_v3m1_base.py:399-421) and its backward.
 * Cluster s is the run [seg_start[s], seg_start[s]+seg_len[s]) of the sorted sequence `order` (int64 rows).
 * out [M,C] and x [N,C] in `dtype`; arg [M,C] int32 = winning source row (first maximum).
 * ------------------------------------------------------------------------------------------- */
int b2pc_segment_max_fwd(const void* x, int dtype, const int64_t* order, const int64_t* seg_start,
                         const int64_t* seg_len, int64_t m, int c, void* out, int32_t* arg, b2pc_stream_t stream);
/* dx [N,C] = scatter of dout [M,C] to the winning rows (dx is zero-filled by the call). */
int b2pc_segment_max_bwd(const void* dout, int dtype, const int32_t* arg, int64_t m, int c, int64_t n, void* dx,
                         b2pc_stream_t stream);

/* Index side of SerializedPooling (point_transformer_v3m1_base.py:371-398) in four small launches and ONE deferred host read:
 * clusters = runs of equal (code[0] >> 3*pooling_depth) in the order-0 sorted sequence.  All outputs are sized for N rows
 * (code_out [n_orders, N] with row stride N); meta[0] = M (clusters), meta[1 + b] = clusters of scene b; the caller reads
 * meta once and slices.  cluster [N] = row -> cluster id; head_pos / head_indices / lengths [M] describe the runs;
 * code_out / batch_out / grid_out are the pooled level's codes (every order), batch ids and grid coordinates (>> depth). */
size_t b2pc_pool_plan_workspace_bytes(int64_t n);
int b2pc_pool_plan(const int64_t* code, int n_orders, int64_t n, const int64_t* order0, const int64_t* batch,
                   const int32_t* grid_coord, int pooling_depth, int n_scene, int64_t* cluster, int64_t* head_pos,
                   int64_t* head_indices, int64_t* lengths, int64_t* code_out, int64_t* batch_out, int32_t* grid_out,
                   int64_t* meta, void* workspace, size_t workspace_bytes, b2pc_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Glue on the path between the two operators (SURVEY.md 8(f).2): fused LayerNorm over point
 * features [N, C] as applied at point_transformer_v3m1_base.py:285,288,300 (nn.LayerNorm under
 * autocast: fp32 statistics).  x / dx in x_dtype, y / dy in y_dtype, gamma/beta/mean/rstd fp32.
 * C in {32, 64, 128, 256, 512} (the PT-v3 widths).
 * ------------------------------------------------------------------------------------------- */
int b2pc_layer_norm_fwd(const void* x, int x_dtype, const float* gamma, const float* beta, int64_t n, int c,
                        float eps, void* y, int y_dtype, float* mean, float* rstd, b2pc_stream_t stream);
size_t b2pc_layer_norm_bwd_workspace_bytes(int64_t n, int c);
int b2pc_layer_norm_bwd(const void* dy, int y_dtype, const void* x, int x_dtype, const float* gamma,
                        const float* mean, const float* rstd, int64_t n, int c, void* dx, float* dgamma,
                        float* dbeta, void* workspace, size_t workspace_bytes, b2pc_stream_t stream);

/* Stochastic depth fused with the residual add (point_transformer_v3m1_base.py:313-334: shortcut + drop_path(x)):
 * out[r, :] = shortcut[r, :] + x[r, :] * rowscale[r]  (out has shortcut's dtype); backward dx[r, :] = dy[r, :] * rowscale[r]. */
int b2pc_rowscale_add(const void* shortcut, int s_dtype, const void* x, int x_dtype, const float* rowscale, int64_t n,
                      int c, void* out, b2pc_stream_t stream);
int b2pc_rowscale(const void* dy, int s_dtype, const float* rowscale, int64_t n, int c, void* dx, int x_dtype,
                  b2pc_stream_t stream);

/* out[c] = sum_r x[r, c] in fp32 (bias gradient of the Linear layers of the block, point_transformer_v3m1_base.py:96-97,
 * 238-240; replaces a tall-matrix torch reduction).  C must be a multiple of 4. */
size_t b2pc_colsum_workspace_bytes(int64_t n, int c);
int b2pc_colsum(const void* x, int dtype, int64_t n, int c, float* out, void* workspace, size_t workspace_bytes,
                b2pc_stream_t stream);


/* ---------------------------------------------------------------------------------------------
 * Serialized attention = patch attention with the reference's [order] gather and [inverse] gather fused in
 * (SerializedAttention.forward, point_transformer_v3m1_base.py:184-216): qkv_points [N, 3, H, D] and out_points [N, H, D]
 * are in POINT order; slot t of the padded patch sequence (T_pad slots, sequences given by cu_seqlens) reads point row
 * gidx[t] = order[pad][t]; sidx[t] = that point row when t is the point's primary slot (inverse = unpad[inverse_order]),
 * and -(r+1) when t is the r-th borrowed filler slot (its output is dropped, :216).  dup_point[r] = the point of filler r.
 * lse [H, T_pad].  Tensor-core path only (head_dim 16, fp16 / bf16): B2PC_ERR_UNSUPPORTED otherwise (callers then run the
 * unfused sequence gather -> b2pc_patch_attn_* -> gather).
 * ------------------------------------------------------------------------------------------- */
int b2pc_serialized_attn_fwd(const void* qkv_points, int dtype, const int32_t* gidx, const int32_t* sidx,
                             const int32_t* cu_seqlens, int n_seq, int max_seqlen, int64_t t_pad, int heads,
                             int head_dim, float scale, void* out_points, float* lse, b2pc_stream_t stream);
size_t b2pc_serialized_attn_bwd_workspace_bytes(int64_t t_pad, int heads, int head_dim, int64_t n_dup);
int b2pc_serialized_attn_bwd(const void* dout_points, const void* qkv_points, const void* out_points, const float* lse,
                             int dtype, const int32_t* gidx, const int32_t* sidx, const int32_t* dup_point,
                             int64_t n_dup, const int32_t* cu_seqlens, int n_seq, int max_seqlen, int64_t t_pad,
                             int heads, int head_dim, float scale, void* dqkv_points, void* workspace,
                             size_t workspace_bytes, b2pc_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Fused residual glue of one PT-v3 block (SURVEY.md 8(f).2; point_transformer_v3m1_base.py:318-338):
 *     t = x;  t = LayerNorm_a(t) [gamma_a != NULL];  t *= (u[row] < keep ? 1/keep : 0) [u != NULL, DropPath :313-315]
 *     r = shortcut + t (fp32, written);  r16 = (dtype) r [r16 != NULL];  y = LayerNorm_b(r) in dtype [gamma_b != NULL]
 * x / r16 / y are `dtype` (fp32, fp16 or bf16), shortcut / r / statistics / affine parameters fp32.
 * stat_a / stat_b: [2, n] (mean, rstd) saved for the backward.  C in {32, 64, 128, 256, 512}.
 * Backward: exact adjoint.  dr_out / dr16 / dy are the gradients of the three outputs (any may be NULL);
 * d_shortcut [n,c] fp32 and dx [n,c] dtype are written; the LayerNorm parameter gradients are reduced deterministically;
 * dx_colsum [c] (optional) receives the column sums of dx = the bias gradient of the Linear that produced x.
 * ------------------------------------------------------------------------------------------- */
int b2pc_fused_residual_fwd(const float* shortcut, const void* x, int dtype, const float* u, float keep,
                            const float* gamma_a, const float* beta_a, float eps_a, const float* gamma_b,
                            const float* beta_b, float eps_b, int64_t n, int c, float* r, void* r16, void* y,
                            float* stat_a, float* stat_b, b2pc_stream_t stream);
size_t b2pc_fused_residual_bwd_workspace_bytes(int64_t n, int c);
int b2pc_fused_residual_bwd(const float* dr_out, const void* dr16, const void* dy, int dtype, const float* r,
                            const void* x, const float* u, float keep, const float* gamma_a, const float* gamma_b,
                            const float* stat_a, const float* stat_b, int64_t n, int c, float* d_shortcut, void* dx,
                            float* dgamma_a, float* dbeta_a, float* dgamma_b, float* dbeta_b, float* dx_colsum,
                            void* workspace, size_t workspace_bytes, b2pc_stream_t stream);

/* One launch refreshes the half-precision shadows of a list of fp32 parameter tensors (what autocast does with one cast
 * kernel per weight per step, torch/amp).  plan: DEVICE array of n_items records {const float* src; void* dst;
 * long long count; long long first_block} with first_block the running sum of ceil(count / 2048); total_blocks its end.
 * dst_dtype B2PC_F16 / B2PC_BF16: cast; B2PC_F32: plain multi-tensor copy (packs the gradients of a parameter list into the
 * flat buffer of the data-parallel all-reduce, the exchange step of pointcept/engines/defaults.py:22-43). */
int b2pc_multi_cast(const void* plan_device, int n_items, long long total_blocks, int dst_dtype, b2pc_stream_t stream);

/* AdamW (torch.optim.AdamW semantics: decoupled weight decay, per-tensor bias correction) over a whole parameter list in one
 * launch.  items: DEVICE array of n_items 56-byte records {float* p; const float* g; float* m; float* v; long long count;
 * long long first_block; float bc1; float bc2_sqrt} with first_block the running sum of ceil(count / 2048), bc1 = 1 - beta1^t and
 * bc2_sqrt = sqrt(1 - beta2^t) for the tensor's own step count t; gradients are multiplied by grad_scale first. */
int b2pc_multi_adamw(const void* items_device, int n_items, long long total_blocks, float lr, float beta1, float beta2, float eps,
                     float weight_decay, float grad_scale, b2pc_stream_t stream);

/* Exact (erf) GELU over n_elems values (n_elems % 4 == 0), forward and backward (nn.GELU, point_transformer_v3m1_base.py:233). */
int b2pc_gelu_fwd(const void* x, int dtype, int64_t n_elems, void* y, b2pc_stream_t stream);
int b2pc_gelu_bwd(const void* dy, const void* x, int dtype, int64_t n_elems, void* dx, b2pc_stream_t stream);
/* GELU backward over [n, c] that also returns colsum[c] = sum_rows dx (fp32): the bias gradient of the Linear feeding the GELU
 * (MLP.fc1, point_transformer_v3m1_base.py:238) without a separate pass over the largest activation of the block. */
size_t b2pc_gelu_bwd_colsum_workspace_bytes(int64_t n, int c);
int b2pc_gelu_bwd_colsum(const void* dy, const void* x, int dtype, int64_t n, int c, void* dx, float* colsum, void* workspace,
                         size_t workspace_bytes, b2pc_stream_t stream);

/* Fused cross-entropy of the segmentation head: nn.CrossEntropyLoss(reduction="mean", ignore_index) on logits [n, n_classes]
 * (pointcept/models/losses/misc.py:13-40, called at pointcept/models/default.py:83-90).  target [n] int64.
 * fwd: lse [n] fp32 (saved for backward), loss_count [2] fp32 = {mean loss over the non-ignored rows, their number};
 * bwd: dlogits = (softmax(logits) - onehot(target)) * grad_loss[0] / count, zero on ignored rows; dlogits has the logits' dtype. */
size_t b2pc_cross_entropy_workspace_bytes(int64_t n);
int b2pc_cross_entropy_fwd(const void* logits, int dtype, const int64_t* target, int64_t n, int n_classes, int64_t ignore_index,
                           float* lse, float* loss_count, void* workspace, size_t workspace_bytes, b2pc_stream_t stream);
int b2pc_cross_entropy_bwd(const void* logits, int dtype, const int64_t* target, const float* lse, const float* grad_loss,
                           const float* loss_count, int64_t n, int n_classes, int64_t ignore_index, void* dlogits,
                           b2pc_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * GPU voxelisation + collate (SURVEY 8(f).3): replaces the per-scene numpy GridSample transform
 * (pointcept/datasets/transform.py:840-958: floor(coord / grid_size), fnv_hash_vec :997-1011 /
 * ravel_hash_vec :980-995, np.argsort, np.unique(return_inverse, return_counts), per-voxel pick)
 * for a whole batch of raw scenes at once, delivering collate_fn's layout
 * (pointcept/datasets/utils.py:19-73: concatenated points + cumulative offset).
 * ------------------------------------------------------------------------------------------- */

/* coord [N,3] fp32 (concatenated raw scenes), offset [B] int64 cumulative raw scene sizes (device), every scene non-empty,
 * max_scene_len = the largest scene (known on the host).  grid_size_host[3] (double).  hash_type 0 = FNV-1a 64, 1 = ravel.
 * math_f64 != 0: coord / grid_size in float64 (NumPy >= 2 promotion of `float32 array / 0-d float64 array`); 0: in float32
 * (NumPy 1.x value-based casting).  Outputs:
 *   grid_coord [N,3] int64   floor(coord / grid) - per-scene minimum          (transform.py:863-866)
 *   inverse    [N]   int64   rank of the point's voxel among the scene's voxels in ascending hash order (:888-890)
 *   sort_index [N]   int64   idx_sort of every scene, concatenated, as global rows (:868; stable order inside a voxel)
 *   vox_start  [N]   int64   first M entries: position in sort_index of each voxel's first member  (cumsum of count, :878)
 *   vox_count  [N]   int64   first M entries: members per voxel (np.unique's count, :870)
 *   meta [1 + 5B] int64: [0] = M; [1..B] = cumulative voxels per scene (the sampled batch's `offset`); [1+B..2B] = count.max()
 *        per scene; [1+2B + 3b + j] = minimum cell of scene b (min_coord = that * grid_size, :867). */
size_t b2pc_grid_sample_workspace_bytes(int64_t n, int batch_size, int64_t max_scene_len);
int b2pc_grid_sample_plan(const float* coord, const int64_t* offset, int batch_size, int64_t n, int64_t max_scene_len,
                          const double* grid_size_host, int hash_type, int math_f64, int64_t* grid_coord, int64_t* inverse,
                          int64_t* sort_index, int64_t* vox_start, int64_t* vox_count, int64_t* meta, void* workspace,
                          size_t workspace_bytes, b2pc_stream_t stream);
/* idx[v] = one member row of voxel v, v < m.  mode 0 (train, transform.py:876-881): member (u % count) with u uniform in
 * [0, count.max()) from a counter-based generator keyed by (arg = seed, v) -- the reference's distribution, modulo bias
 * included; mode 1 (test, :914-916): member (arg % count), arg = fragment number. */
int b2pc_grid_sample_select(const int64_t* sort_index, const int64_t* vox_start, const int64_t* vox_count, const int64_t* meta,
                            int batch_size, int64_t m, int mode, uint64_t arg, int64_t* idx, b2pc_stream_t stream);
/* displacement[v, :] = (coord[idx[v]] / grid - min) - grid_coord - 0.5 (transform.py:893-895); out_f64 selects the output type */
int b2pc_grid_sample_displacement(const float* coord, const int64_t* idx, const int64_t* meta, int batch_size, int64_t m,
                                  const double* grid_size_host, int math_f64, void* out, int out_f64, b2pc_stream_t stream);
/* dst[i, :] = src[idx[i], :], rows of row_bytes bytes of any payload type: index_operator (transform.py:24-40) for every
 * per-point key of the batch in the sampled order. */
int b2pc_gather_rows(const void* src, int64_t row_bytes, const int64_t* idx, int64_t m, void* dst, b2pc_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Variants sharing the kernels (SURVEY 8(f).4): evaluation-time operators and PointROPE.
 * ------------------------------------------------------------------------------------------- */

/* pointops.knn_query (libs/pointops/functions/query.py:7-26, src/knn_query/knn_query_cuda_kernel.cu:60-104): for every query
 * new_xyz[i] of scene b the nsample nearest points of xyz inside the same scene, ascending.  xyz [n,3], new_xyz [m,3] fp32,
 * offset / new_offset [B] int32 cumulative.  idx [m,nsample] int32 (-1 = fewer than nsample points), dist2 [m,nsample] squared
 * distances (1e10 placeholder); the Python surface returns sqrt(dist2) as the reference does.  1 <= nsample <= 128. */
int b2pc_knn_query(const float* xyz, const int32_t* offset, const float* new_xyz, const int32_t* new_offset, int batch_size,
                   int64_t m, int nsample, int32_t* idx, float* dist2, b2pc_stream_t stream);
/* Fragment voting of the tester (pointcept/engines/test.py:193-203): pred[index[i], :] += softmax(logits[i, :]).
 * logits [n, n_classes] (dtype enum), index [n] int64, pred [*, n_classes] fp32. */
int b2pc_vote_accumulate(const void* logits, int dtype, const int64_t* index, int64_t n, int n_classes, float* pred,
                         b2pc_stream_t stream);
/* PointROPE (libs/pointrope/kernels.cu:19-103; litept_v1.py:29-59): in-place rotary embedding of n_heads heads of head_dim
 * channels per token with integer positions pos [n_tokens,3] int64; fwd = +F0 forward, -F0 backward (the rotation's inverse).
 * token_stride (elements) lets the packed qkv [T,3,H,D] be rotated in place: tokens = qkv, token_stride = 3*H*D, n_heads = 2*H
 * rotates q and k and leaves v.  head_dim % 6 == 0. */
int b2pc_point_rope(void* tokens, int dtype, const int64_t* pos, int64_t n_tokens, int64_t token_stride, int n_heads,
                    int head_dim, float base, float fwd, b2pc_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Built-in per-entry-point timing (bench.py's roofline leg; binding independent because it lives below the C ABI).
 * While enabled, every hot entry point brackets its kernels with a CUDA-event pair on the caller's stream and records the
 * ALGORITHMIC work of the call (SURVEY.md 8(d): compulsory bytes, and flops where the host knows them).
 * b2pc_profile_collect synchronises the recorded events and aggregates per entry point.
 * ------------------------------------------------------------------------------------------- */
enum {
  B2PC_P_ATTN_FWD = 0, B2PC_P_ATTN_BWD = 1, B2PC_P_CONV = 2, B2PC_P_WGRAD = 3, B2PC_P_ENCODE = 4, B2PC_P_SORT = 5,
  B2PC_P_RULEBOOK_SUBM = 6, B2PC_P_RULEBOOK_STRIDED = 7, B2PC_P_PADDING = 8, B2PC_P_FUSED_RESIDUAL = 9, B2PC_P_LAYER_NORM = 10,
  B2PC_P_SEGMENT_MAX = 11, B2PC_P_COLSUM = 12, B2PC_P_OTHER = 13, B2PC_P_COUNT = 14
};
typedef struct { int id; long long calls; double ms; double flops; double bytes; } b2pc_profile_entry;
void b2pc_profile_enable(int on);                           /* on != 0: clear the records and start; 0: stop */
int b2pc_profile_collect(b2pc_profile_entry* out, int max_entries);   /* returns the number of entries written (<= B2PC_P_COUNT) */

#ifdef __cplusplus
}
#endif
#endif /* B2PC_H_ */
