// libb2pc.so -- C ABI (include/b2pc.h) over the sm_90a kernels.  No torch types cross this boundary.
#include <stdarg.h>

#include "common.cuh"
#include "serialize.cuh"
#include "sort.cuh"
#include "rulebook.cuh"
#include "spconv_simt.cuh"
#include "attn_simt.cuh"
#include "layernorm.cuh"
#include "fused.cuh"
#include "pool.cuh"
#include "voxelize.cuh"
#include "eval_ops.cuh"
#include "loss.cuh"
#include "attn_mma.cuh"
#include "spconv_mma.cuh"

#include <atomic>
#include <mutex>
#include <vector>

namespace b2pc {
static std::atomic<long long> g_launches{0};
void count_launches(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace b2pc

using namespace b2pc;

// ---- built-in timing of the entry points (b2pc_profile_*) ------------------------------------------------------------------
namespace {
struct ProfRec { int id; cudaEvent_t e0, e1; double flops, bytes; };
std::atomic<bool> g_prof_on{false};
std::mutex g_prof_mu;
std::vector<ProfRec> g_prof;
struct ProfScope {
  cudaStream_t s; int id; double flops, bytes; cudaEvent_t e0{nullptr};
  ProfScope(b2pc_stream_t stream, int id_, double fl, double by) : s((cudaStream_t)stream), id(id_), flops(fl), bytes(by) {
    if (g_prof_on.load(std::memory_order_relaxed)) { cudaEventCreate(&e0); cudaEventRecord(e0, s); }
  }
  ~ProfScope() {
    if (!e0) return;
    cudaEvent_t e1;
    cudaEventCreate(&e1);
    cudaEventRecord(e1, s);
    std::lock_guard<std::mutex> lk(g_prof_mu);
    g_prof.push_back(ProfRec{id, e0, e1, flops, bytes});
  }
};
}  // namespace
#define B2PC_PROF(stream, id, flops, bytes) ProfScope prof_scope__((stream), (id), (double)(flops), (double)(bytes))

extern "C" {

int b2pc_version(void) { return 100; }
const char* b2pc_last_error(void) { return g_err; }
long long b2pc_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

int b2pc_serialize_encode(const int32_t* grid_coord, const int64_t* batch, int64_t n, int depth, const int* orders_host,
                          int n_orders, int64_t* code, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_ENCODE, 0, (double)n * (20.0 + 8.0 * n_orders));
  B2PC_CHECK_ARG(grid_coord && code && orders_host, "serialize_encode: null pointer");
  return launch_encode(grid_coord, batch, n, depth, orders_host, n_orders, code, (cudaStream_t)stream);
}

size_t b2pc_serialize_sort_workspace_bytes(int64_t n, int n_orders) { return sort_workspace_bytes(n, n_orders); }

int b2pc_serialize_sort(const int64_t* code, int64_t n, int n_orders, int key_bits, int64_t* order, int64_t* inverse,
                        void* workspace, size_t workspace_bytes, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_SORT, 0, (double)n * n_orders * ((key_bits + 7) / 8) * 24.0);
  B2PC_CHECK_ARG(code && order && inverse && workspace, "serialize_sort: null pointer");
  return launch_sort(code, n, n_orders, key_bits, order, inverse, workspace, workspace_bytes, (cudaStream_t)stream);
}

int b2pc_patch_padding(const int64_t* offset, int batch_size, int patch_size, int64_t n, int64_t t_pad, int n_seq,
                       int64_t* pad, int64_t* unpad, int32_t* cu_seqlens, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_PADDING, 0, 8.0 * t_pad + 8.0 * n);
  B2PC_CHECK_ARG(offset && pad && unpad && cu_seqlens, "patch_padding: null pointer");
  return launch_padding(offset, batch_size, patch_size, n, t_pad, n_seq, pad, unpad, cu_seqlens, (cudaStream_t)stream);
}

// ---- attention ------------------------------------------------------------------------------------
int b2pc_patch_attn_fwd(const void* qkv, int dtype, const int32_t* cu_seqlens, int n_seq, int max_seqlen, int64_t t,
                        int heads, int head_dim, float scale, void* out, float* lse, int impl, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_ATTN_FWD, 4.0 * t * max_seqlen * heads * head_dim, 16.0 * t * heads * head_dim);
  B2PC_CHECK_ARG(qkv && cu_seqlens && out && lse, "patch_attn_fwd: null pointer");
  B2PC_CHECK_ARG(dtype == B2PC_F16 || dtype == B2PC_BF16, "patch_attn_fwd: dtype must be fp16 or bf16 (got %d)", dtype);
  B2PC_CHECK_ARG(n_seq >= 0 && max_seqlen >= 0 && t >= 0 && heads > 0 && head_dim > 0, "patch_attn_fwd: bad sizes");
  cudaStream_t s = (cudaStream_t)stream;
  if (impl != 1) {
    if (attn_mma_supported(dtype, head_dim)) return launch_attn_fwd_mma(qkv, dtype, cu_seqlens, n_seq, max_seqlen, t, heads, head_dim, scale, out, lse, s);
    if (impl == 2) { set_error("patch_attn_fwd: tensor-core kernel does not support dtype %d head_dim %d", dtype, head_dim); return B2PC_ERR_UNSUPPORTED; }
  }
  if (dtype == B2PC_F16) return launch_attn_fwd_simt<__half>(qkv, cu_seqlens, n_seq, max_seqlen, t, heads, head_dim, scale, out, lse, s);
  return launch_attn_fwd_simt<__nv_bfloat16>(qkv, cu_seqlens, n_seq, max_seqlen, t, heads, head_dim, scale, out, lse, s);
}

size_t b2pc_patch_attn_bwd_workspace_bytes(int64_t t, int heads, int head_dim) {
  size_t b = attn_bwd_workspace_bytes(t, heads, head_dim);
  size_t u = attn_bwd_mma_workspace_bytes(t, heads, head_dim);
  if (u > b) b = u;
  return b;
}

int b2pc_patch_attn_bwd(const void* dout, const void* qkv, const void* out, const float* lse, int dtype,
                        const int32_t* cu_seqlens, int n_seq, int max_seqlen, int64_t t, int heads, int head_dim,
                        float scale, void* dqkv, void* workspace, size_t workspace_bytes, int impl, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_ATTN_BWD, 10.0 * t * max_seqlen * heads * head_dim, 32.0 * t * heads * head_dim);
  B2PC_CHECK_ARG(dout && qkv && out && lse && cu_seqlens && dqkv && workspace, "patch_attn_bwd: null pointer");
  B2PC_CHECK_ARG(dtype == B2PC_F16 || dtype == B2PC_BF16, "patch_attn_bwd: dtype must be fp16 or bf16 (got %d)", dtype);
  if (workspace_bytes < b2pc_patch_attn_bwd_workspace_bytes(t, heads, head_dim)) { set_error("patch_attn_bwd: workspace too small"); return B2PC_ERR_WORKSPACE; }
  cudaStream_t s = (cudaStream_t)stream;
  if (impl != 1) {
    if (attn_mma_supported(dtype, head_dim)) return launch_attn_bwd_mma(dout, qkv, out, lse, dtype, cu_seqlens, n_seq, max_seqlen, t, heads, head_dim, scale, dqkv, workspace, s);
    if (impl == 2) { set_error("patch_attn_bwd: tensor-core kernel does not support dtype %d head_dim %d", dtype, head_dim); return B2PC_ERR_UNSUPPORTED; }
  }
  if (dtype == B2PC_F16) return launch_attn_bwd_simt<__half>(dout, qkv, out, lse, cu_seqlens, n_seq, max_seqlen, t, heads, head_dim, scale, dqkv, workspace, s);
  return launch_attn_bwd_simt<__nv_bfloat16>(dout, qkv, out, lse, cu_seqlens, n_seq, max_seqlen, t, heads, head_dim, scale, dqkv, workspace, s);
}

// ---- rulebooks --------------------------------------------------------------------------------------
size_t b2pc_rulebook_workspace_bytes(int64_t n, int reach) { return rulebook_workspace_bytes(n, reach); }
size_t b2pc_rulebook_strided_workspace_bytes(int64_t n, const int* ksize_host, const int* stride_host, const int* dilation_host) {
  if (!ksize_host) return 0;
  return rulebook_workspace_bytes(n, strided_reach(ksize_host, stride_host, dilation_host));
}

int b2pc_rulebook_subm(const int32_t* indices, int64_t n, const int* spatial_shape_host, const int* ksize_host,
                       const int* dilation_host, int32_t* pair, void* workspace, size_t workspace_bytes, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_RULEBOOK_SUBM, 0, (double)n * (16.0 + 4.0 * ksize_host[0] * ksize_host[1] * ksize_host[2]));
  B2PC_CHECK_ARG(indices && spatial_shape_host && ksize_host && pair && workspace, "rulebook_subm: null pointer");
  return launch_rulebook_subm(indices, n, spatial_shape_host, ksize_host, dilation_host, pair, workspace, workspace_bytes, (cudaStream_t)stream);
}

int b2pc_rulebook_strided_begin(const int32_t* indices, int64_t n, const int* spatial_shape_host, const int* ksize_host,
                                const int* stride_host, const int* padding_host, const int* dilation_host, int64_t* num_out,
                                void* workspace, size_t workspace_bytes, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_RULEBOOK_STRIDED, 0, 16.0 * n);
  B2PC_CHECK_ARG(indices && spatial_shape_host && ksize_host && num_out && workspace, "rulebook_strided_begin: null pointer");
  return launch_rulebook_strided_begin(indices, n, spatial_shape_host, ksize_host, stride_host, padding_host, dilation_host, num_out, workspace, workspace_bytes, (cudaStream_t)stream);
}

int b2pc_rulebook_strided_finish(const int32_t* indices, int64_t n, const int* spatial_shape_host, const int* ksize_host,
                                 const int* stride_host, const int* padding_host, const int* dilation_host, int64_t num_out_host,
                                 int batch_count_host, int32_t* out_indices, int32_t* pair_fwd, int32_t* pair_bwd, void* workspace, size_t workspace_bytes,
                                 b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_RULEBOOK_STRIDED, 0, (double)(n + num_out_host) * (16.0 + 4.0 * ksize_host[0] * ksize_host[1] * ksize_host[2]));
  B2PC_CHECK_ARG(indices && spatial_shape_host && ksize_host && out_indices && pair_fwd && pair_bwd && workspace, "rulebook_strided_finish: null pointer");
  return launch_rulebook_strided_finish(indices, n, spatial_shape_host, ksize_host, stride_host, padding_host, dilation_host, num_out_host, batch_count_host, out_indices, pair_fwd, pair_bwd, workspace, workspace_bytes, (cudaStream_t)stream);
}

// ---- sparse convolution arithmetic ---------------------------------------------------------------------
size_t b2pc_spconv_gather_gemm_workspace_bytes(int64_t n_out, int c_in, int c_out, int kv) {
  return conv_mma_workspace_bytes(n_out, c_in, c_out, kv);
}

int b2pc_spconv_gather_gemm(const void* feat, const void* weight, const void* bias, const int32_t* pair, int64_t pair_stride,
                            int64_t n_in, int64_t n_out, int c_in, int c_out, int kv, int transpose_w, int flip, int dtype,
                            void* out, void* workspace, size_t workspace_bytes, int impl, b2pc_stream_t stream) {
  const double es__ = dtype == B2PC_F32 ? 4.0 : 2.0;
  B2PC_PROF(stream, B2PC_P_CONV, 0, es__ * ((double)n_in * c_in + (double)n_out * c_out + (double)kv * c_in * c_out) + 4.0 * kv * n_out);
  B2PC_CHECK_ARG(feat && weight && pair && out, "spconv_gather_gemm: null pointer");
  B2PC_CHECK_ARG(n_in >= 0 && n_out >= 0 && c_in > 0 && c_out > 0 && kv > 0 && pair_stride >= n_out, "spconv_gather_gemm: bad sizes");
  cudaStream_t s = (cudaStream_t)stream;
  if (impl != 1) {
    if (spconv_mma_supported(dtype, c_in, c_out)) {
      const size_t need = conv_mma_workspace_bytes(n_out, c_in, c_out, kv);
      if (!workspace || workspace_bytes < need) { set_error("spconv_gather_gemm: workspace too small"); return B2PC_ERR_WORKSPACE; }
      return launch_gather_gemm_mma(feat, weight, bias, pair, pair_stride, n_out, c_in, c_out, kv, transpose_w, flip, dtype, out, workspace, s);
    }
    if (impl == 2) { set_error("spconv_gather_gemm: tensor-core kernel does not support dtype %d c_in %d c_out %d", dtype, c_in, c_out); return B2PC_ERR_UNSUPPORTED; }
  }
  switch (dtype) {
    case B2PC_F32: return launch_gather_gemm_simt<float>(feat, weight, bias, pair, pair_stride, n_out, c_in, c_out, kv, transpose_w, flip, out, s);
    case B2PC_F16: return launch_gather_gemm_simt<__half>(feat, weight, bias, pair, pair_stride, n_out, c_in, c_out, kv, transpose_w, flip, out, s);
    case B2PC_BF16: return launch_gather_gemm_simt<__nv_bfloat16>(feat, weight, bias, pair, pair_stride, n_out, c_in, c_out, kv, transpose_w, flip, out, s);
  }
  set_error("spconv_gather_gemm: unknown dtype %d", dtype);
  return B2PC_ERR_INVALID_ARG;
}

size_t b2pc_spconv_bwd_weight_workspace_bytes(int64_t n_out, int c_in, int c_out, int kv) {
  size_t b = bwd_weight_workspace_bytes(n_out, c_in, c_out, kv);
  size_t u = wgrad_mma_workspace_bytes(n_out, c_in, c_out, kv);
  if (u > b) b = u;
  return b;
}

int b2pc_spconv_bwd_weight(const void* feat_in, const void* dout, const int32_t* pair, int64_t pair_stride, int64_t n_in,
                           int64_t n_out, int c_in, int c_out, int kv, int dtype, float* dweight, void* workspace,
                           size_t workspace_bytes, int impl, b2pc_stream_t stream) {
  const double es__ = dtype == B2PC_F32 ? 4.0 : 2.0;
  B2PC_PROF(stream, B2PC_P_WGRAD, 0, es__ * ((double)n_in * c_in + (double)n_out * c_out) + 4.0 * kv * n_out + 4.0 * kv * c_in * c_out);
  B2PC_CHECK_ARG(feat_in && dout && pair && dweight && workspace, "spconv_bwd_weight: null pointer");
  B2PC_CHECK_ARG(n_in >= 0 && n_out >= 0 && c_in > 0 && c_out > 0 && kv > 0 && pair_stride >= n_out, "spconv_bwd_weight: bad sizes");
  cudaStream_t s = (cudaStream_t)stream;
  if (workspace_bytes < b2pc_spconv_bwd_weight_workspace_bytes(n_out, c_in, c_out, kv)) { set_error("spconv_bwd_weight: workspace too small"); return B2PC_ERR_WORKSPACE; }
  if (impl != 1 && n_out > 0) {
    if (wgrad_mma_supported(dtype, c_in, c_out)) return launch_bwd_weight_mma(feat_in, dout, pair, pair_stride, n_out, c_in, c_out, kv, dtype, dweight, workspace, s);
    if (impl == 2) { set_error("spconv_bwd_weight: tensor-core kernel does not support dtype %d c_in %d c_out %d", dtype, c_in, c_out); return B2PC_ERR_UNSUPPORTED; }
  }
  switch (dtype) {
    case B2PC_F32: return launch_bwd_weight_simt<float>(feat_in, dout, pair, pair_stride, n_out, c_in, c_out, kv, dweight, workspace, workspace_bytes, s);
    case B2PC_F16: return launch_bwd_weight_simt<__half>(feat_in, dout, pair, pair_stride, n_out, c_in, c_out, kv, dweight, workspace, workspace_bytes, s);
    case B2PC_BF16: return launch_bwd_weight_simt<__nv_bfloat16>(feat_in, dout, pair, pair_stride, n_out, c_in, c_out, kv, dweight, workspace, workspace_bytes, s);
  }
  set_error("spconv_bwd_weight: unknown dtype %d", dtype);
  return B2PC_ERR_INVALID_ARG;
}

// ---- serialized pooling (segment max over runs of the sorted order) --------------------------------------------------------
int b2pc_segment_max_fwd(const void* x, int dtype, const int64_t* order, const int64_t* seg_start, const int64_t* seg_len, int64_t m,
                         int c, void* out, int32_t* arg, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_SEGMENT_MAX, 0, 0);
  B2PC_CHECK_ARG(x && order && seg_start && seg_len && out && arg, "segment_max_fwd: null pointer");
  B2PC_CHECK_ARG(m >= 0 && c > 0, "segment_max_fwd: bad sizes");
  return launch_segment_max_fwd(x, dtype, order, seg_start, seg_len, m, c, out, arg, (cudaStream_t)stream);
}

int b2pc_segment_max_bwd(const void* dout, int dtype, const int32_t* arg, int64_t m, int c, int64_t n, void* dx, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_SEGMENT_MAX, 0, 0);
  B2PC_CHECK_ARG(dout && arg && dx, "segment_max_bwd: null pointer");
  B2PC_CHECK_ARG(m >= 0 && c > 0 && n >= 0, "segment_max_bwd: bad sizes");
  return launch_segment_max_bwd(dout, dtype, arg, m, c, n, dx, (cudaStream_t)stream);
}

size_t b2pc_pool_plan_workspace_bytes(int64_t n) { return pool_plan_workspace_bytes(n); }

int b2pc_pool_plan(const int64_t* code, int n_orders, int64_t n, const int64_t* order0, const int64_t* batch, const int32_t* grid_coord,
                   int pooling_depth, int n_scene, int64_t* cluster, int64_t* head_pos, int64_t* head_indices, int64_t* lengths,
                   int64_t* code_out, int64_t* batch_out, int32_t* grid_out, int64_t* meta, void* workspace, size_t workspace_bytes,
                   b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_OTHER, 0, 0);
  B2PC_CHECK_ARG(code && order0 && batch && grid_coord && cluster && head_pos && head_indices && lengths && code_out && batch_out &&
                 grid_out && meta && workspace, "pool_plan: null pointer");
  return launch_pool_plan(code, n_orders, n, order0, batch, grid_coord, pooling_depth, n_scene, cluster, head_pos, head_indices, lengths,
                          code_out, batch_out, grid_out, meta, workspace, workspace_bytes, (cudaStream_t)stream);
}

// ---- glue: fused LayerNorm ---------------------------------------------------------------------------------------
int b2pc_layer_norm_fwd(const void* x, int x_dtype, const float* gamma, const float* beta, int64_t n, int c, float eps, void* y,
                        int y_dtype, float* mean, float* rstd, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_LAYER_NORM, 0, (double)n * c * 6.0);
  B2PC_CHECK_ARG(x && gamma && y && mean && rstd, "layer_norm_fwd: null pointer");
  return launch_layer_norm_fwd(x, x_dtype, gamma, beta, n, c, eps, y, y_dtype, mean, rstd, (cudaStream_t)stream);
}

size_t b2pc_layer_norm_bwd_workspace_bytes(int64_t n, int c) { return layer_norm_bwd_workspace_bytes(n, c); }

int b2pc_layer_norm_bwd(const void* dy, int y_dtype, const void* x, int x_dtype, const float* gamma, const float* mean,
                        const float* rstd, int64_t n, int c, void* dx, float* dgamma, float* dbeta, void* workspace,
                        size_t workspace_bytes, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_LAYER_NORM, 0, (double)n * c * 8.0);
  B2PC_CHECK_ARG(dy && x && gamma && mean && rstd && dx && dgamma && workspace, "layer_norm_bwd: null pointer");
  return launch_layer_norm_bwd(dy, y_dtype, x, x_dtype, gamma, mean, rstd, n, c, dx, dgamma, dbeta, workspace, workspace_bytes,
                               (cudaStream_t)stream);
}

int b2pc_rowscale_add(const void* shortcut, int s_dtype, const void* x, int x_dtype, const float* rowscale, int64_t n, int c, void* out,
                      b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_OTHER, 0, 0);
  B2PC_CHECK_ARG(shortcut && x && rowscale && out, "rowscale_add: null pointer");
  return launch_rowscale_add(shortcut, s_dtype, x, x_dtype, rowscale, n, c, out, (cudaStream_t)stream);
}

int b2pc_rowscale(const void* dy, int s_dtype, const float* rowscale, int64_t n, int c, void* dx, int x_dtype, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_OTHER, 0, 0);
  B2PC_CHECK_ARG(dy && rowscale && dx, "rowscale: null pointer");
  return launch_rowscale(dy, s_dtype, rowscale, n, c, dx, x_dtype, (cudaStream_t)stream);
}

size_t b2pc_colsum_workspace_bytes(int64_t n, int c) { return colsum_workspace_bytes(n, c); }

int b2pc_colsum(const void* x, int dtype, int64_t n, int c, float* out, void* workspace, size_t workspace_bytes, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_COLSUM, 0, (double)n * c * (dtype == B2PC_F32 ? 4.0 : 2.0));
  B2PC_CHECK_ARG(x && out && workspace, "colsum: null pointer");
  return launch_colsum(x, dtype, n, c, out, workspace, workspace_bytes, (cudaStream_t)stream);
}

// ---- serialized attention (gather-fused patch attention) -----------------------------------------------------------------
int b2pc_serialized_attn_fwd(const void* qkv_points, int dtype, const int32_t* gidx, const int32_t* sidx, const int32_t* cu_seqlens,
                             int n_seq, int max_seqlen, int64_t t_pad, int heads, int head_dim, float scale, void* out_points,
                             float* lse, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_ATTN_FWD, 4.0 * t_pad * max_seqlen * heads * head_dim, 16.0 * t_pad * heads * head_dim);
  B2PC_CHECK_ARG(qkv_points && gidx && sidx && cu_seqlens && out_points && lse, "serialized_attn_fwd: null pointer");
  B2PC_CHECK_ARG(n_seq >= 0 && max_seqlen >= 0 && t_pad >= 0 && heads > 0 && head_dim > 0, "serialized_attn_fwd: bad sizes");
  if (attn_mma_supported(dtype, head_dim))
    return launch_attn_fwd_mma(qkv_points, dtype, cu_seqlens, n_seq, max_seqlen, t_pad, heads, head_dim, scale, out_points, lse,
                               (cudaStream_t)stream, gidx, sidx);
  set_error("serialized_attn_fwd: needs the tensor-core kernel (fp16/bf16, head_dim 16); got dtype %d head_dim %d", dtype, head_dim);
  return B2PC_ERR_UNSUPPORTED;
}

size_t b2pc_serialized_attn_bwd_workspace_bytes(int64_t t_pad, int heads, int head_dim, int64_t n_dup) {
  return attn_bwd_mma_workspace_bytes(t_pad, heads, head_dim, n_dup);
}

int b2pc_serialized_attn_bwd(const void* dout_points, const void* qkv_points, const void* out_points, const float* lse, int dtype,
                             const int32_t* gidx, const int32_t* sidx, const int32_t* dup_point, int64_t n_dup,
                             const int32_t* cu_seqlens, int n_seq, int max_seqlen, int64_t t_pad, int heads, int head_dim, float scale,
                             void* dqkv_points, void* workspace, size_t workspace_bytes, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_ATTN_BWD, 10.0 * t_pad * max_seqlen * heads * head_dim, 32.0 * t_pad * heads * head_dim);
  B2PC_CHECK_ARG(dout_points && qkv_points && out_points && lse && gidx && sidx && cu_seqlens && dqkv_points && workspace,
                 "serialized_attn_bwd: null pointer");
  B2PC_CHECK_ARG(n_dup == 0 || dup_point, "serialized_attn_bwd: dup_point missing");
  if (attn_mma_supported(dtype, head_dim)) {
    if (workspace_bytes < attn_bwd_mma_workspace_bytes(t_pad, heads, head_dim, n_dup)) { set_error("serialized_attn_bwd: workspace too small"); return B2PC_ERR_WORKSPACE; }
    return launch_attn_bwd_mma(dout_points, qkv_points, out_points, lse, dtype, cu_seqlens, n_seq, max_seqlen, t_pad, heads, head_dim, scale,
                               dqkv_points, workspace, (cudaStream_t)stream, gidx, sidx, dup_point, n_dup);
  }
  set_error("serialized_attn_bwd: needs the tensor-core kernel (fp16/bf16, head_dim 16); got dtype %d head_dim %d", dtype, head_dim);
  return B2PC_ERR_UNSUPPORTED;
}

// ---- fused residual glue ------------------------------------------------------------------------------------------------
int b2pc_fused_residual_fwd(const float* shortcut, const void* x, int dtype, const float* u, float keep, const float* gamma_a,
                            const float* beta_a, float eps_a, const float* gamma_b, const float* beta_b, float eps_b, int64_t n, int c,
                            float* r, void* r16, void* y, float* stat_a, float* stat_b, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_FUSED_RESIDUAL, 0, (double)n * c * (8.0 + (dtype == B2PC_F32 ? 4.0 : 2.0) * (1 + (r16 != nullptr) + (y != nullptr))));
  FusedResArgs a{shortcut, x, u, keep, gamma_a, beta_a, gamma_b, beta_b, eps_a, eps_b, n, c, r, r16, y, stat_a, stat_b};
  return launch_fused_residual_fwd(a, dtype, (cudaStream_t)stream);
}

size_t b2pc_fused_residual_bwd_workspace_bytes(int64_t n, int c) { return fused_residual_bwd_workspace_bytes(n, c); }

int b2pc_fused_residual_bwd(const float* dr_out, const void* dr16, const void* dy, int dtype, const float* r, const void* x,
                            const float* u, float keep, const float* gamma_a, const float* gamma_b, const float* stat_a,
                            const float* stat_b, int64_t n, int c, float* d_shortcut, void* dx, float* dgamma_a, float* dbeta_a,
                            float* dgamma_b, float* dbeta_b, float* dx_colsum, void* workspace, size_t workspace_bytes,
                            b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_FUSED_RESIDUAL, 0, (double)n * c * (12.0 + (dtype == B2PC_F32 ? 4.0 : 2.0) * (2 + (dr16 != nullptr) + (dy != nullptr))));
  FusedResBwdArgs a{dr_out, dr16, dy, r, x, u, keep, gamma_a, gamma_b, stat_a, stat_b, n, c, d_shortcut, dx, nullptr, 0};
  return launch_fused_residual_bwd(a, dtype, dgamma_a, dbeta_a, dgamma_b, dbeta_b, dx_colsum, workspace, workspace_bytes, (cudaStream_t)stream);
}

int b2pc_multi_cast(const void* plan_device, int n_items, long long total_blocks, int dst_dtype, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_OTHER, 0, 0);
  return launch_multi_cast(plan_device, n_items, total_blocks, dst_dtype, (cudaStream_t)stream);
}

int b2pc_multi_adamw(const void* items_device, int n_items, long long total_blocks, float lr, float beta1, float beta2, float eps,
                     float weight_decay, float grad_scale, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_OTHER, 0, 0);
  return launch_multi_adamw(items_device, n_items, total_blocks, lr, beta1, beta2, eps, weight_decay, grad_scale, (cudaStream_t)stream);
}

static int gelu_grid(int64_t total4) {
  int64_t b = ceil_div(total4 > 0 ? total4 : 1, 256);
  return (int)(b > kNumSMs * 16 ? kNumSMs * 16 : b);
}

int b2pc_gelu_fwd(const void* x, int dtype, int64_t n_elems, void* y, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_OTHER, 0, 0);
  B2PC_CHECK_ARG(x && y && n_elems >= 0 && n_elems % 4 == 0, "gelu_fwd: bad arguments");
  if (n_elems == 0) return B2PC_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t t4 = n_elems / 4;
  switch (dtype) {
    case B2PC_F32: gelu_fwd_kernel<float><<<gelu_grid(t4), 256, 0, s>>>((const float*)x, t4, (float*)y); break;
    case B2PC_F16: gelu_fwd_kernel<__half><<<gelu_grid(t4), 256, 0, s>>>((const __half*)x, t4, (__half*)y); break;
    case B2PC_BF16: gelu_fwd_kernel<__nv_bfloat16><<<gelu_grid(t4), 256, 0, s>>>((const __nv_bfloat16*)x, t4, (__nv_bfloat16*)y); break;
    default: set_error("gelu_fwd: unknown dtype %d", dtype); return B2PC_ERR_INVALID_ARG;
  }
  count_launches(1);
  B2PC_CHECK_LAUNCH("gelu_fwd");
  return B2PC_OK;
}

int b2pc_gelu_bwd(const void* dy, const void* x, int dtype, int64_t n_elems, void* dx, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_OTHER, 0, 0);
  B2PC_CHECK_ARG(dy && x && dx && n_elems >= 0 && n_elems % 4 == 0, "gelu_bwd: bad arguments");
  if (n_elems == 0) return B2PC_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t t4 = n_elems / 4;
  switch (dtype) {
    case B2PC_F32: gelu_bwd_kernel<float><<<gelu_grid(t4), 256, 0, s>>>((const float*)dy, (const float*)x, t4, (float*)dx); break;
    case B2PC_F16: gelu_bwd_kernel<__half><<<gelu_grid(t4), 256, 0, s>>>((const __half*)dy, (const __half*)x, t4, (__half*)dx); break;
    case B2PC_BF16: gelu_bwd_kernel<__nv_bfloat16><<<gelu_grid(t4), 256, 0, s>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x, t4, (__nv_bfloat16*)dx); break;
    default: set_error("gelu_bwd: unknown dtype %d", dtype); return B2PC_ERR_INVALID_ARG;
  }
  count_launches(1);
  B2PC_CHECK_LAUNCH("gelu_bwd");
  return B2PC_OK;
}

size_t b2pc_gelu_bwd_colsum_workspace_bytes(int64_t n, int c) { return gelu_bwd_colsum_workspace_bytes(n, c); }

int b2pc_gelu_bwd_colsum(const void* dy, const void* x, int dtype, int64_t n, int c, void* dx, float* colsum, void* workspace,
                         size_t workspace_bytes, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_OTHER, 0, 0);
  B2PC_CHECK_ARG(dy && x && dx && colsum && workspace, "gelu_bwd_colsum: null pointer");
  return launch_gelu_bwd_colsum(dy, x, dtype, n, c, dx, colsum, workspace, workspace_bytes, (cudaStream_t)stream);
}

// ---- fused cross-entropy ------------------------------------------------------------------------------------------------------
size_t b2pc_cross_entropy_workspace_bytes(int64_t n) { return cross_entropy_workspace_bytes(n); }

int b2pc_cross_entropy_fwd(const void* logits, int dtype, const int64_t* target, int64_t n, int n_classes, int64_t ignore_index, float* lse,
                           float* loss_count, void* workspace, size_t workspace_bytes, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_OTHER, 0, (double)n * (n_classes * (dtype == B2PC_F32 ? 4 : 2) + 12));
  B2PC_CHECK_ARG(logits && target && lse && loss_count && workspace, "cross_entropy_fwd: null pointer");
  B2PC_CHECK_ARG(n > 0 && n_classes >= 1 && dtype >= 0 && dtype <= 2, "cross_entropy_fwd: bad arguments");
  if (workspace_bytes < cross_entropy_workspace_bytes(n)) { set_error("cross_entropy_fwd: workspace too small"); return B2PC_ERR_WORKSPACE; }
  cudaStream_t s = (cudaStream_t)stream;
  const int blocks = ce_blocks(n);
  float* partial = (float*)workspace;
  if (dtype == B2PC_F32) cross_entropy_fwd_kernel<float><<<blocks, kCeThreads, 0, s>>>((const float*)logits, target, n, n_classes, ignore_index, lse, partial);
  else if (dtype == B2PC_F16) cross_entropy_fwd_kernel<__half><<<blocks, kCeThreads, 0, s>>>((const __half*)logits, target, n, n_classes, ignore_index, lse, partial);
  else cross_entropy_fwd_kernel<__nv_bfloat16><<<blocks, kCeThreads, 0, s>>>((const __nv_bfloat16*)logits, target, n, n_classes, ignore_index, lse, partial);
  cross_entropy_finish_kernel<<<1, 32, 0, s>>>(partial, blocks, loss_count);
  count_launches(2);
  B2PC_CHECK_LAUNCH("cross_entropy_fwd");
  return B2PC_OK;
}

int b2pc_cross_entropy_bwd(const void* logits, int dtype, const int64_t* target, const float* lse, const float* grad_loss, const float* loss_count,
                           int64_t n, int n_classes, int64_t ignore_index, void* dlogits, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_OTHER, 0, (double)n * (2.0 * n_classes * (dtype == B2PC_F32 ? 4 : 2) + 12));
  B2PC_CHECK_ARG(logits && target && lse && grad_loss && loss_count && dlogits, "cross_entropy_bwd: null pointer");
  B2PC_CHECK_ARG(n > 0 && n_classes >= 1 && dtype >= 0 && dtype <= 2, "cross_entropy_bwd: bad arguments");
  cudaStream_t s = (cudaStream_t)stream;
  int64_t b = ceil_div(n * n_classes, kCeThreads);
  if (b > kNumSMs * 16) b = kNumSMs * 16;
  if (dtype == B2PC_F32) cross_entropy_bwd_kernel<float><<<(unsigned)b, kCeThreads, 0, s>>>((const float*)logits, target, lse, grad_loss, loss_count, n, n_classes, ignore_index, (float*)dlogits);
  else if (dtype == B2PC_F16) cross_entropy_bwd_kernel<__half><<<(unsigned)b, kCeThreads, 0, s>>>((const __half*)logits, target, lse, grad_loss, loss_count, n, n_classes, ignore_index, (__half*)dlogits);
  else cross_entropy_bwd_kernel<__nv_bfloat16><<<(unsigned)b, kCeThreads, 0, s>>>((const __nv_bfloat16*)logits, target, lse, grad_loss, loss_count, n, n_classes, ignore_index, (__nv_bfloat16*)dlogits);
  count_launches(1);
  B2PC_CHECK_LAUNCH("cross_entropy_bwd");
  return B2PC_OK;
}

// ---- GPU voxelisation / collate (SURVEY 8(f).3) -----------------------------------------------------------------------------
size_t b2pc_grid_sample_workspace_bytes(int64_t n, int batch_size, int64_t max_scene_len) {
  if (n <= 0 || batch_size <= 0 || max_scene_len <= 0) return 256;
  return grid_sample_workspace_bytes(n, batch_size, max_scene_len);
}

int b2pc_grid_sample_plan(const float* coord, const int64_t* offset, int batch_size, int64_t n, int64_t max_scene_len,
                          const double* grid_size_host, int hash_type, int math_f64, int64_t* grid_coord, int64_t* inverse,
                          int64_t* sort_index, int64_t* vox_start, int64_t* vox_count, int64_t* meta, void* workspace,
                          size_t workspace_bytes, b2pc_stream_t stream) {
  B2PC_PROF(stream, B2PC_P_OTHER, 0, (double)n * (12.0 + 24.0 + 8.0 * 24.0 + 40.0));
  B2PC_CHECK_ARG(coord && offset && grid_size_host && grid_coord && inverse && sort_index && vox_start && vox_count && meta && workspace,
                 "grid_sample_plan: null pointer");
  return launch_grid_sample_plan(coord, offset, batch_size, n, max_scene_len, grid_size_host, hash_type, math_f64, grid_coord, inverse,
                                 sort_index, vox_start, vox_count, meta, workspace, workspace_bytes, (cudaStream_t)stream);
}

int b2pc_grid_sample_select(const int64_t* sort_index, const int64_t* vox_start, const int64_t* vox_count, const int64_t* meta,
                            int batch_size, int64_t m, int mode, uint64_t arg, int64_t* idx, b2pc_stream_t stream) {
  B2PC_CHECK_ARG(sort_index && vox_start && vox_count && meta && idx, "grid_sample_select: null pointer");
  B2PC_CHECK_ARG(m >= 0 && batch_size >= 1 && (mode == 0 || mode == 1), "grid_sample_select: bad arguments");
  if (m == 0) return B2PC_OK;
  gs_select_kernel<<<(unsigned)ceil_div(m, kGsThreads), kGsThreads, 0, (cudaStream_t)stream>>>(sort_index, vox_start, vox_count, meta,
                                                                                             batch_size, m, mode, arg, idx);
  count_launches(1);
  B2PC_CHECK_LAUNCH("grid_sample_select");
  return B2PC_OK;
}

int b2pc_grid_sample_displacement(const float* coord, const int64_t* idx, const int64_t* meta, int batch_size, int64_t m,
                                  const double* grid_size_host, int math_f64, void* out, int out_f64, b2pc_stream_t stream) {
  B2PC_CHECK_ARG(coord && idx && meta && grid_size_host && out, "grid_sample_displacement: null pointer");
  B2PC_CHECK_ARG(m >= 0 && batch_size >= 1, "grid_sample_displacement: bad sizes");
  if (m == 0) return B2PC_OK;
  GsGrid gg;
  for (int j = 0; j < 3; ++j) { gg.g[j] = grid_size_host[j]; gg.gf[j] = (float)grid_size_host[j]; }
  const unsigned blocks = (unsigned)ceil_div(m, kGsThreads);
  cudaStream_t s = (cudaStream_t)stream;
  if (math_f64 && out_f64) gs_displacement_kernel<true, double><<<blocks, kGsThreads, 0, s>>>(coord, idx, meta, batch_size, m, gg, (double*)out);
  else if (math_f64) gs_displacement_kernel<true, float><<<blocks, kGsThreads, 0, s>>>(coord, idx, meta, batch_size, m, gg, (float*)out);
  else if (out_f64) gs_displacement_kernel<false, double><<<blocks, kGsThreads, 0, s>>>(coord, idx, meta, batch_size, m, gg, (double*)out);
  else gs_displacement_kernel<false, float><<<blocks, kGsThreads, 0, s>>>(coord, idx, meta, batch_size, m, gg, (float*)out);
  count_launches(1);
  B2PC_CHECK_LAUNCH("grid_sample_displacement");
  return B2PC_OK;
}

int b2pc_gather_rows(const void* src, int64_t row_bytes, const int64_t* idx, int64_t m, void* dst, b2pc_stream_t stream) {
  B2PC_CHECK_ARG(src && idx && dst, "gather_rows: null pointer");
  B2PC_CHECK_ARG(row_bytes > 0 && m >= 0, "gather_rows: bad sizes");
  if (m == 0) return B2PC_OK;
  cudaStream_t s = (cudaStream_t)stream;
  const uintptr_t al = (uintptr_t)src | (uintptr_t)dst | (uintptr_t)row_bytes;
  auto blocks = [&](int64_t vecs) { int64_t b = ceil_div(m * vecs, kGsThreads); return (unsigned)(b > kNumSMs * 16 ? kNumSMs * 16 : b); };
  if (al % 16 == 0) gather_rows_kernel<uint4><<<blocks(row_bytes / 16), kGsThreads, 0, s>>>((const uint4*)src, row_bytes / 16, idx, m, (uint4*)dst);
  else if (al % 8 == 0) gather_rows_kernel<uint2><<<blocks(row_bytes / 8), kGsThreads, 0, s>>>((const uint2*)src, row_bytes / 8, idx, m, (uint2*)dst);
  else if (al % 4 == 0) gather_rows_kernel<uint32_t><<<blocks(row_bytes / 4), kGsThreads, 0, s>>>((const uint32_t*)src, row_bytes / 4, idx, m, (uint32_t*)dst);
  else gather_rows_kernel<uint8_t><<<blocks(row_bytes), kGsThreads, 0, s>>>((const uint8_t*)src, row_bytes, idx, m, (uint8_t*)dst);
  count_launches(1);
  B2PC_CHECK_LAUNCH("gather_rows");
  return B2PC_OK;
}

// ---- variants sharing the kernels (SURVEY 8(f).4) ----------------------------------------------------------------------------
int b2pc_knn_query(const float* xyz, const int32_t* offset, const float* new_xyz, const int32_t* new_offset, int batch_size, int64_t m,
                   int nsample, int32_t* idx, float* dist2, b2pc_stream_t stream) {
  B2PC_CHECK_ARG(xyz && offset && new_xyz && new_offset && idx && dist2, "knn_query: null pointer");
  return launch_knn_query(xyz, offset, new_xyz, new_offset, batch_size, m, nsample, idx, dist2, (cudaStream_t)stream);
}

int b2pc_vote_accumulate(const void* logits, int dtype, const int64_t* index, int64_t n, int n_classes, float* pred, b2pc_stream_t stream) {
  B2PC_CHECK_ARG(logits && index && pred, "vote_accumulate: null pointer");
  B2PC_CHECK_ARG(n >= 0 && n_classes >= 1 && dtype >= 0 && dtype <= 2, "vote_accumulate: bad arguments");
  if (n == 0) return B2PC_OK;
  const unsigned blocks = (unsigned)ceil_div(n * 32, 256);
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype == B2PC_F32) vote_accumulate_kernel<float><<<blocks, 256, 0, s>>>((const float*)logits, index, n, n_classes, pred);
  else if (dtype == B2PC_F16) vote_accumulate_kernel<__half><<<blocks, 256, 0, s>>>((const __half*)logits, index, n, n_classes, pred);
  else vote_accumulate_kernel<__nv_bfloat16><<<blocks, 256, 0, s>>>((const __nv_bfloat16*)logits, index, n, n_classes, pred);
  count_launches(1);
  B2PC_CHECK_LAUNCH("vote_accumulate");
  return B2PC_OK;
}

int b2pc_point_rope(void* tokens, int dtype, const int64_t* pos, int64_t n_tokens, int64_t token_stride, int n_heads, int head_dim, float base,
                    float fwd, b2pc_stream_t stream) {
  B2PC_CHECK_ARG(tokens && pos, "point_rope: null pointer");
  B2PC_CHECK_ARG(head_dim > 0 && head_dim % 6 == 0, "point_rope: token dim must be multiple of 6 (got %d)", head_dim);
  B2PC_CHECK_ARG(n_tokens >= 0 && n_heads >= 1 && token_stride >= (int64_t)n_heads * head_dim && dtype >= 0 && dtype <= 2, "point_rope: bad arguments");
  if (n_tokens == 0) return B2PC_OK;
  const unsigned blocks = (unsigned)ceil_div(n_tokens * (head_dim / 2), 256);
  cudaStream_t s = (cudaStream_t)stream;
  if (dtype == B2PC_F32) point_rope_kernel<float><<<blocks, 256, 0, s>>>((float*)tokens, pos, n_tokens, token_stride, n_heads, head_dim, base, fwd);
  else if (dtype == B2PC_F16) point_rope_kernel<__half><<<blocks, 256, 0, s>>>((__half*)tokens, pos, n_tokens, token_stride, n_heads, head_dim, base, fwd);
  else point_rope_kernel<__nv_bfloat16><<<blocks, 256, 0, s>>>((__nv_bfloat16*)tokens, pos, n_tokens, token_stride, n_heads, head_dim, base, fwd);
  count_launches(1);
  B2PC_CHECK_LAUNCH("point_rope");
  return B2PC_OK;
}

void b2pc_profile_enable(int on) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  if (on) {
    for (auto& r : g_prof) { cudaEventDestroy(r.e0); cudaEventDestroy(r.e1); }
    g_prof.clear();
  }
  g_prof_on.store(on != 0);
}

int b2pc_profile_collect(b2pc_profile_entry* out, int max_entries) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  b2pc_profile_entry agg[B2PC_P_COUNT];
  for (int i = 0; i < B2PC_P_COUNT; ++i) agg[i] = b2pc_profile_entry{i, 0, 0.0, 0.0, 0.0};
  for (auto& r : g_prof) {
    float ms = 0.f;
    if (cudaEventSynchronize(r.e1) == cudaSuccess && cudaEventElapsedTime(&ms, r.e0, r.e1) == cudaSuccess && r.id >= 0 && r.id < B2PC_P_COUNT) {
      agg[r.id].calls += 1; agg[r.id].ms += ms; agg[r.id].flops += r.flops; agg[r.id].bytes += r.bytes;
    }
    cudaEventDestroy(r.e0);
    cudaEventDestroy(r.e1);
  }
  g_prof.clear();
  int n = 0;
  for (int i = 0; i < B2PC_P_COUNT && n < max_entries; ++i)
    if (agg[i].calls > 0) out[n++] = agg[i];
  return n;
}

}  // extern "C"
