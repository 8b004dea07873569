// SIMT patch attention (one thread per query / per key, fp32 math): the always-available correctness
// path and the on-GPU A/B reference for the tensor-core kernels in attn_mma.cuh.
// Layouts follow flash_attn_varlen_qkvpacked_func: qkv [T,3,H,D], out [T,H,D], lse [H,T] (natural log).
#pragma once
#include "common.cuh"

namespace b2pc {

constexpr int kAsQ = 128;   // queries (threads) per block
constexpr int kAsKV = 64;   // keys staged per tile
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;

template <typename T, int D>
__global__ void __launch_bounds__(kAsQ)
attn_fwd_simt_kernel(const T* __restrict__ qkv, const int32_t* __restrict__ cu, int64_t t_total, int H, float scale,
                     T* __restrict__ out, float* __restrict__ lse) {
  __shared__ float Ks[kAsKV][D];
  __shared__ float Vs[kAsKV][D];
  const int seq = blockIdx.x, h = blockIdx.z;
  const int64_t s0 = cu[seq], s1 = cu[seq + 1];
  const int len = (int)(s1 - s0);
  const int q0 = blockIdx.y * kAsQ;
  if (q0 >= len) return;
  const int qi = q0 + threadIdx.x;
  const bool qok = qi < len;
  const float sc2 = scale * kLog2e;
  float q[D], o[D];
#pragma unroll
  for (int d = 0; d < D; ++d) { q[d] = qok ? to_f32(qkv[(((s0 + qi) * 3 + 0) * H + h) * D + d]) * sc2 : 0.f; o[d] = 0.f; }
  float m = -INFINITY, l = 0.f;
  for (int k0 = 0; k0 < len; k0 += kAsKV) {
    const int nk = min(kAsKV, len - k0);
    __syncthreads();
    for (int e = threadIdx.x; e < kAsKV * D; e += kAsQ) {
      const int r = e / D, d = e % D;
      float kv = 0.f, vv = 0.f;
      if (r < nk) {
        kv = to_f32(qkv[(((s0 + k0 + r) * 3 + 1) * H + h) * D + d]);
        vv = to_f32(qkv[(((s0 + k0 + r) * 3 + 2) * H + h) * D + d]);
      }
      Ks[r][d] = kv; Vs[r][d] = vv;
    }
    __syncthreads();
    for (int j0 = 0; j0 < nk; j0 += 8) {
      float s[8];
      float cm = -INFINITY;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        float a = 0.f;
#pragma unroll
        for (int d = 0; d < D; ++d) a = fmaf(q[d], Ks[j0 + jj][d], a);
        s[jj] = (j0 + jj < nk) ? a : -INFINITY;
        cm = fmaxf(cm, s[jj]);
      }
      const float mn = fmaxf(m, cm);
      const float corr = exp2f(m - mn);
      l *= corr;
#pragma unroll
      for (int d = 0; d < D; ++d) o[d] *= corr;
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const float p = exp2f(s[jj] - mn);
        l += p;
#pragma unroll
        for (int d = 0; d < D; ++d) o[d] = fmaf(p, Vs[j0 + jj][d], o[d]);
      }
      m = mn;
    }
  }
  if (qok) {
    const float inv = 1.f / l;
#pragma unroll
    for (int d = 0; d < D; ++d) out[((s0 + qi) * H + h) * D + d] = from_f32<T>(o[d] * inv);
    lse[(int64_t)h * t_total + s0 + qi] = (m + log2f(l)) * kLn2;
  }
}

// delta[h, t] = sum_d dout[t,h,d] * out[t,h,d]
template <typename T>
__global__ void __launch_bounds__(256)
attn_delta_kernel(const T* __restrict__ dout, const T* __restrict__ out, int64_t t_total, int H, int D,
                  float* __restrict__ delta) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;  // over T*H
  if (i >= t_total * H) return;
  const int64_t t = i / H; const int h = (int)(i % H);
  float a = 0.f;
  for (int d = 0; d < D; ++d) a = fmaf(to_f32(dout[i * D + d]), to_f32(out[i * D + d]), a);
  delta[(int64_t)h * t_total + t] = a;
}

template <typename T, int D>
__global__ void __launch_bounds__(kAsQ)
attn_bwd_dq_simt_kernel(const T* __restrict__ dout, const T* __restrict__ qkv, const float* __restrict__ lse,
                        const float* __restrict__ delta, const int32_t* __restrict__ cu, int64_t t_total, int H,
                        float scale, T* __restrict__ dqkv) {
  __shared__ float Ks[kAsKV][D];
  __shared__ float Vs[kAsKV][D];
  const int seq = blockIdx.x, h = blockIdx.z;
  const int64_t s0 = cu[seq], s1 = cu[seq + 1];
  const int len = (int)(s1 - s0);
  const int q0 = blockIdx.y * kAsQ;
  if (q0 >= len) return;
  const int qi = q0 + threadIdx.x;
  const bool qok = qi < len;
  const float sc2 = scale * kLog2e;
  float q[D], g[D], dq[D];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    q[d] = qok ? to_f32(qkv[(((s0 + qi) * 3 + 0) * H + h) * D + d]) * sc2 : 0.f;
    g[d] = qok ? to_f32(dout[((s0 + qi) * H + h) * D + d]) : 0.f;
    dq[d] = 0.f;
  }
  const float l2 = qok ? lse[(int64_t)h * t_total + s0 + qi] * kLog2e : 0.f;
  const float dl = qok ? delta[(int64_t)h * t_total + s0 + qi] : 0.f;
  for (int k0 = 0; k0 < len; k0 += kAsKV) {
    const int nk = min(kAsKV, len - k0);
    __syncthreads();
    for (int e = threadIdx.x; e < kAsKV * D; e += kAsQ) {
      const int r = e / D, d = e % D;
      float kv = 0.f, vv = 0.f;
      if (r < nk) {
        kv = to_f32(qkv[(((s0 + k0 + r) * 3 + 1) * H + h) * D + d]);
        vv = to_f32(qkv[(((s0 + k0 + r) * 3 + 2) * H + h) * D + d]);
      }
      Ks[r][d] = kv; Vs[r][d] = vv;
    }
    __syncthreads();
    for (int j = 0; j < nk; ++j) {
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int d = 0; d < D; ++d) { s = fmaf(q[d], Ks[j][d], s); dp = fmaf(g[d], Vs[j][d], dp); }
      const float p = exp2f(s - l2);
      const float ds = p * (dp - dl);
#pragma unroll
      for (int d = 0; d < D; ++d) dq[d] = fmaf(ds, Ks[j][d], dq[d]);
    }
  }
  if (qok) {
#pragma unroll
    for (int d = 0; d < D; ++d) dqkv[(((s0 + qi) * 3 + 0) * H + h) * D + d] = from_f32<T>(dq[d] * scale);
  }
}

template <typename T, int D>
__global__ void __launch_bounds__(kAsQ)
attn_bwd_dkv_simt_kernel(const T* __restrict__ dout, const T* __restrict__ qkv, const float* __restrict__ lse,
                         const float* __restrict__ delta, const int32_t* __restrict__ cu, int64_t t_total, int H,
                         float scale, T* __restrict__ dqkv) {
  __shared__ float Qs[kAsKV][D];
  __shared__ float Gs[kAsKV][D];
  __shared__ float Ls[kAsKV], Dl[kAsKV];
  const int seq = blockIdx.x, h = blockIdx.z;
  const int64_t s0 = cu[seq], s1 = cu[seq + 1];
  const int len = (int)(s1 - s0);
  const int kbase = blockIdx.y * kAsQ;
  if (kbase >= len) return;
  const int ki = kbase + threadIdx.x;
  const bool kok = ki < len;
  const float sc2 = scale * kLog2e;
  float kk[D], vv[D], dk[D], dv[D];
#pragma unroll
  for (int d = 0; d < D; ++d) {
    kk[d] = kok ? to_f32(qkv[(((s0 + ki) * 3 + 1) * H + h) * D + d]) : 0.f;
    vv[d] = kok ? to_f32(qkv[(((s0 + ki) * 3 + 2) * H + h) * D + d]) : 0.f;
    dk[d] = 0.f; dv[d] = 0.f;
  }
  for (int q0 = 0; q0 < len; q0 += kAsKV) {
    const int nq = min(kAsKV, len - q0);
    __syncthreads();
    for (int e = threadIdx.x; e < kAsKV * D; e += kAsQ) {
      const int r = e / D, d = e % D;
      float qv = 0.f, gv = 0.f;
      if (r < nq) {
        qv = to_f32(qkv[(((s0 + q0 + r) * 3 + 0) * H + h) * D + d]) * sc2;
        gv = to_f32(dout[((s0 + q0 + r) * H + h) * D + d]);
      }
      Qs[r][d] = qv; Gs[r][d] = gv;
    }
    if (threadIdx.x < kAsKV) {
      const int r = threadIdx.x;
      Ls[r] = r < nq ? lse[(int64_t)h * t_total + s0 + q0 + r] * kLog2e : 0.f;
      Dl[r] = r < nq ? delta[(int64_t)h * t_total + s0 + q0 + r] : 0.f;
    }
    __syncthreads();
    for (int i = 0; i < nq; ++i) {
      float s = 0.f, dp = 0.f;
#pragma unroll
      for (int d = 0; d < D; ++d) { s = fmaf(Qs[i][d], kk[d], s); dp = fmaf(Gs[i][d], vv[d], dp); }
      const float p = exp2f(s - Ls[i]);
      const float ds = p * (dp - Dl[i]);
#pragma unroll
      for (int d = 0; d < D; ++d) { dv[d] = fmaf(p, Gs[i][d], dv[d]); dk[d] = fmaf(ds, Qs[i][d], dk[d]); }
    }
  }
  if (kok) {
    // Qs was pre-multiplied by scale*log2e: dk accumulated ds * q * scale * log2e -> divide log2e back out
    const float fix = 1.f / kLog2e;
#pragma unroll
    for (int d = 0; d < D; ++d) {
      dqkv[(((s0 + ki) * 3 + 1) * H + h) * D + d] = from_f32<T>(dk[d] * fix);
      dqkv[(((s0 + ki) * 3 + 2) * H + h) * D + d] = from_f32<T>(dv[d]);
    }
  }
}

template <typename T>
inline int launch_attn_fwd_simt(const void* qkv, const int32_t* cu, int n_seq, int max_seqlen, int64_t t, int H, int D,
                                float scale, void* out, float* lse, cudaStream_t stream) {
  if (n_seq == 0 || t == 0) return B2PC_OK;
  dim3 grid(n_seq, (unsigned)ceil_div(max_seqlen, kAsQ), H);
#define B2PC_AF(DD) attn_fwd_simt_kernel<T, DD><<<grid, kAsQ, 0, stream>>>((const T*)qkv, cu, t, H, scale, (T*)out, lse)
  switch (D) {
    case 8: B2PC_AF(8); break;
    case 16: B2PC_AF(16); break;
    case 18: B2PC_AF(18); break;   // LitePT / PT-v3m3 RoPE heads (litept_v1.py, head_dim 18)
    case 24: B2PC_AF(24); break;
    case 32: B2PC_AF(32); break;
    case 48: B2PC_AF(48); break;
    case 64: B2PC_AF(64); break;
    default: set_error("patch_attn_fwd(simt): head_dim %d not in {8,16,18,24,32,48,64}", D); return B2PC_ERR_UNSUPPORTED;
  }
#undef B2PC_AF
  count_launches(1);
  B2PC_CHECK_LAUNCH("patch_attn_fwd(simt)");
  return B2PC_OK;
}

inline size_t attn_bwd_workspace_bytes(int64_t t, int H, int D) {
  (void)D;
  return align_up((size_t)t * H * sizeof(float), 256) * 2 + (size_t)t * H * 4 * sizeof(float) * 0 + 256;
}

template <typename T>
inline int launch_attn_bwd_simt(const void* dout, const void* qkv, const void* out, const float* lse, const int32_t* cu,
                                int n_seq, int max_seqlen, int64_t t, int H, int D, float scale, void* dqkv, void* ws,
                                cudaStream_t stream) {
  if (n_seq == 0 || t == 0) return B2PC_OK;
  float* delta = (float*)ws;
  attn_delta_kernel<T><<<(unsigned)ceil_div(t * H, 256), 256, 0, stream>>>((const T*)dout, (const T*)out, t, H, D, delta);
  dim3 grid(n_seq, (unsigned)ceil_div(max_seqlen, kAsQ), H);
#define B2PC_AB(DD)                                                                                                         \
  attn_bwd_dq_simt_kernel<T, DD><<<grid, kAsQ, 0, stream>>>((const T*)dout, (const T*)qkv, lse, delta, cu, t, H, scale, (T*)dqkv); \
  attn_bwd_dkv_simt_kernel<T, DD><<<grid, kAsQ, 0, stream>>>((const T*)dout, (const T*)qkv, lse, delta, cu, t, H, scale, (T*)dqkv)
  switch (D) {
    case 8: B2PC_AB(8); break;
    case 16: B2PC_AB(16); break;
    case 18: B2PC_AB(18); break;
    case 24: B2PC_AB(24); break;
    case 32: B2PC_AB(32); break;
    case 48: B2PC_AB(48); break;
    case 64: B2PC_AB(64); break;
    default: set_error("patch_attn_bwd(simt): head_dim %d not in {8,16,18,24,32,48,64}", D); return B2PC_ERR_UNSUPPORTED;
  }
#undef B2PC_AB
  count_launches(3);
  B2PC_CHECK_LAUNCH("patch_attn_bwd(simt)");
  return B2PC_OK;
}

}  // namespace b2pc
