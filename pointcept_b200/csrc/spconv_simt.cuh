// SIMT (CUDA-core, fp32 accumulate) sparse-convolution kernels: the always-available correctness path
// and the on-GPU A/B reference for the tensor-core kernels in spconv_mma.cuh.
#pragma once
#include "common.cuh"

namespace b2pc {

constexpr int kCgTileM = 64, kCgTileN = 64, kCgTileK = 32;

// out[j, n] = bias[n] + sum_k sum_c in[pair[k', j], c] * W_k(c, n)
template <typename T>
__global__ void __launch_bounds__(256)
gather_gemm_simt_kernel(const T* __restrict__ feat, const T* __restrict__ weight, const T* __restrict__ bias,
                        const int32_t* __restrict__ pair, int64_t pair_stride, int64_t n_out, int c_in, int c_out,
                        int kv, int transpose_w, int flip, T* __restrict__ out) {
  __shared__ float As[kCgTileK][kCgTileM + 4];
  __shared__ float Ws[kCgTileK][kCgTileN + 4];
  __shared__ int32_t idx[kCgTileM];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t row0 = (int64_t)blockIdx.x * kCgTileM;
  const int col0 = blockIdx.y * kCgTileN;
  float acc[4][4] = {};
  for (int k = 0; k < kv; ++k) {
    const int kp = flip ? kv - 1 - k : k;
    int any = 0;
    if (tid < kCgTileM) {
      const int64_t j = row0 + tid;
      const int32_t v = (j < n_out) ? pair[(int64_t)kp * pair_stride + j] : -1;
      idx[tid] = v;
      any = v >= 0;
    }
    if (!__syncthreads_or(any)) continue;
    for (int c0 = 0; c0 < c_in; c0 += kCgTileK) {
      // gather A: 64 rows x 32 channels; a warp reads 32 consecutive channels of one row
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        const int r = it * 8 + (tid >> 5), c = tid & 31;
        const int32_t src = idx[r];
        float v = 0.f;
        if (src >= 0 && c0 + c < c_in) v = to_f32(feat[(int64_t)src * c_in + c0 + c]);
        As[c][r] = v;
      }
      // W tile: 32 (c) x 64 (n)
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        int c, n;
        if (transpose_w) { n = tid & 63; c = it * 4 + (tid >> 6); }   // weight[(c*kv+k)*c_out + n]: n contiguous
        else { c = tid & 31; n = it * 8 + (tid >> 5); }              // weight[(n*kv+k)*c_in + c]: c contiguous
        float v = 0.f;
        if (c0 + c < c_in && col0 + n < c_out)
          v = transpose_w ? to_f32(weight[((int64_t)(c0 + c) * kv + k) * c_out + col0 + n])
                          : to_f32(weight[((int64_t)(col0 + n) * kv + k) * c_in + c0 + c]);
        Ws[c][n] = v;
      }
      __syncthreads();
#pragma unroll 8
      for (int c = 0; c < kCgTileK; ++c) {
        const float4 a = *reinterpret_cast<const float4*>(&As[c][ty * 4]);
        const float4 b = *reinterpret_cast<const float4*>(&Ws[c][tx * 4]);
        const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t j = row0 + ty * 4 + i;
    if (j >= n_out) continue;
#pragma unroll
    for (int jj = 0; jj < 4; ++jj) {
      const int n = col0 + tx * 4 + jj;
      if (n < c_out) out[j * c_out + n] = from_f32<T>(acc[i][jj] + (bias ? to_f32(bias[n]) : 0.f));
    }
  }
}

template <typename T>
inline int launch_gather_gemm_simt(const void* feat, const void* weight, const void* bias, const int32_t* pair,
                                   int64_t pair_stride, int64_t n_out, int c_in, int c_out, int kv, int transpose_w,
                                   int flip, void* out, cudaStream_t stream) {
  if (n_out == 0) return B2PC_OK;
  dim3 grid((unsigned)ceil_div(n_out, kCgTileM), (unsigned)ceil_div(c_out, kCgTileN));
  gather_gemm_simt_kernel<T><<<grid, 256, 0, stream>>>((const T*)feat, (const T*)weight, (const T*)bias, pair, pair_stride,
                                                       n_out, c_in, c_out, kv, transpose_w, flip, (T*)out);
  count_launches(1);
  B2PC_CHECK_LAUNCH("spconv_gather_gemm(simt)");
  return B2PC_OK;
}

// ---- weight gradient ------------------------------------------------------------------------------
// partial[s][co][k][ci] = sum over the rows of split s of dout[j, co] * feat[pair[k, j], ci]
constexpr int kWgRows = 64, kWgCi = 32, kWgCo = 64;

inline int bwd_weight_splits(int64_t n_out) {
  int64_t s = ceil_div(n_out, (int64_t)kWgRows * 8);
  return (int)(s < 1 ? 1 : (s > 64 ? 64 : s));
}

template <typename T>
__global__ void __launch_bounds__(256)
bwd_weight_simt_kernel(const T* __restrict__ feat, const T* __restrict__ dout, const int32_t* __restrict__ pair,
                       int64_t pair_stride, int64_t n_out, int c_in, int c_out, int kv, int splits,
                       float* __restrict__ partial) {
  __shared__ float Fs[kWgRows][kWgCi + 1];
  __shared__ float Ds[kWgRows][kWgCo + 4];
  __shared__ int32_t idx[kWgRows];
  const int k = blockIdx.x;
  const int n_ci_tiles = (c_in + kWgCi - 1) / kWgCi;
  const int ci0 = (blockIdx.y % n_ci_tiles) * kWgCi;
  const int co0 = (blockIdx.y / n_ci_tiles) * kWgCo;
  const int split = blockIdx.z;
  const int tid = threadIdx.x;
  // thread -> 2 ci x 4 co
  const int tci = (tid & 15) * 2, tco = (tid >> 4) * 4;
  float acc[2][4] = {};
  const int64_t rows_per_split = ceil_div(ceil_div(n_out, splits), kWgRows) * kWgRows;
  const int64_t r_begin = split * rows_per_split;
  int64_t r_end = r_begin + rows_per_split;
  if (r_end > n_out) r_end = n_out;
  for (int64_t r0 = r_begin; r0 < r_end; r0 += kWgRows) {
    int any = 0;
    if (tid < kWgRows) {
      const int64_t j = r0 + tid;
      const int32_t v = (j < r_end) ? pair[(int64_t)k * pair_stride + j] : -1;
      idx[tid] = v;
      any = v >= 0;
    }
    if (!__syncthreads_or(any)) continue;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      const int r = it * 8 + (tid >> 5), c = tid & 31;
      const int32_t src = idx[r];
      Fs[r][c] = (src >= 0 && ci0 + c < c_in) ? to_f32(feat[(int64_t)src * c_in + ci0 + c]) : 0.f;
    }
#pragma unroll
    for (int it = 0; it < 16; ++it) {
      const int r = it * 4 + (tid >> 6), c = tid & 63;
      const int64_t j = r0 + r;
      Ds[r][c] = (idx[r] >= 0 && co0 + c < c_out) ? to_f32(dout[j * c_out + co0 + c]) : 0.f;
    }
    __syncthreads();
#pragma unroll 8
    for (int r = 0; r < kWgRows; ++r) {
      const float f0 = Fs[r][tci], f1 = Fs[r][tci + 1];
      const float4 d = *reinterpret_cast<const float4*>(&Ds[r][tco]);
      acc[0][0] = fmaf(f0, d.x, acc[0][0]); acc[0][1] = fmaf(f0, d.y, acc[0][1]);
      acc[0][2] = fmaf(f0, d.z, acc[0][2]); acc[0][3] = fmaf(f0, d.w, acc[0][3]);
      acc[1][0] = fmaf(f1, d.x, acc[1][0]); acc[1][1] = fmaf(f1, d.y, acc[1][1]);
      acc[1][2] = fmaf(f1, d.z, acc[1][2]); acc[1][3] = fmaf(f1, d.w, acc[1][3]);
    }
    __syncthreads();
  }
  float* p = partial + (int64_t)split * c_out * kv * c_in;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int ci = ci0 + tci + i, co = co0 + tco + j;
      if (ci < c_in && co < c_out) p[((int64_t)co * kv + k) * c_in + ci] = acc[i][j];
    }
}

__global__ void __launch_bounds__(256)
reduce_splits_kernel(const float* __restrict__ partial, int64_t elems, int splits, float* __restrict__ out) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < elems; i += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int sp = 0; sp < splits; ++sp) s += partial[(int64_t)sp * elems + i];
    out[i] = s;
  }
}

inline size_t bwd_weight_workspace_bytes(int64_t n_out, int c_in, int c_out, int kv) {
  return (size_t)bwd_weight_splits(n_out) * c_out * kv * c_in * sizeof(float) + 256;
}

template <typename T>
inline int launch_bwd_weight_simt(const void* feat, const void* dout, const int32_t* pair, int64_t pair_stride,
                                  int64_t n_out, int c_in, int c_out, int kv, float* dweight, void* ws, size_t ws_bytes,
                                  cudaStream_t stream) {
  const int64_t elems = (int64_t)c_out * kv * c_in;
  if (n_out == 0) { cudaMemsetAsync(dweight, 0, elems * sizeof(float), stream); return B2PC_OK; }
  if (ws_bytes < bwd_weight_workspace_bytes(n_out, c_in, c_out, kv)) { set_error("spconv_bwd_weight: workspace too small"); return B2PC_ERR_WORKSPACE; }
  const int splits = bwd_weight_splits(n_out);
  const int n_ci = (c_in + kWgCi - 1) / kWgCi, n_co = (c_out + kWgCo - 1) / kWgCo;
  dim3 grid(kv, n_ci * n_co, splits);
  bwd_weight_simt_kernel<T><<<grid, 256, 0, stream>>>((const T*)feat, (const T*)dout, pair, pair_stride, n_out, c_in, c_out,
                                                      kv, splits, (float*)ws);
  int rb = (int)ceil_div(elems, 256); if (rb > kNumSMs * 8) rb = kNumSMs * 8;
  reduce_splits_kernel<<<rb, 256, 0, stream>>>((const float*)ws, elems, splits, dweight);
  count_launches(2);
  B2PC_CHECK_LAUNCH("spconv_bwd_weight(simt)");
  return B2PC_OK;
}

}  // namespace b2pc
