// Sparse convolution on the Hopper tensor cores (mma.sync m16n8k16, fp16 / bf16 in, fp32 accumulate in registers).
//
// Forward / backward-data: output-stationary implicit GEMM
//   out[j, :] = bias + sum_k  feat[pair[k', j], :] @ W_k            (k' = flip ? KV-1-k : k)
// One CTA owns 128 consecutive output rows x NT output channels (four warps, 32 rows each); the accumulator stays in registers for
// the whole sweep over kernel offsets.  Per unit = (active offset k, channel chunk of KC): thread t gathers row pair[k', row0+t]
// (zero-filled when the pair is absent) with cp.async, the matching K-major W_k slice is staged next to it, and every warp runs
// KC/16 x 2 x NT/8 MMAs from ldmatrix fragments.  Offsets with no partner in the whole tile are skipped.  A 3-stage ring keeps two
// units in flight while the tensor cores work on a third.  Shared-memory rows are padded by 16 bytes so that the eight rows an
// ldmatrix phase reads fall on distinct bank groups.
// Every output element is written once.  When the launch is under-filled (deep levels) the offsets are split over several CTAs per
// tile; each split stores its fp32 partial tile to its own slice of a scratch buffer and a small kernel sums the slices in a fixed
// order (deterministic).
#pragma once
#include "common.cuh"
#include "mma.cuh"
#include "spconv_simt.cuh"   // reduce_splits_kernel

namespace b2pc {

constexpr int kCmM = 128;       // output rows per CTA
constexpr int kCmMaxKV = 32;    // kernel offsets per rulebook chunk staged in shared memory (27 for 3^3, 125 for 5^3 in four chunks)
constexpr int kCmStages = 3;    // ring depth

template <int KC, int NT> __host__ __device__ constexpr int conv_mma_stage_bytes() { return (kCmM + NT) * (KC * 2 + 16); }
template <int KC, int NT> __host__ __device__ constexpr int conv_mma_smem_bytes() {
  return kCmMaxKV * kCmM * 4 + 128 + kCmStages * conv_mma_stage_bytes<KC, NT>();
}

struct ConvMmaCfg { int kc, n_tile, ksplit; };

inline ConvMmaCfg conv_mma_cfg(int64_t n_out, int c_in, int c_out, int kv) {
  ConvMmaCfg c;
  c.kc = c_in % 32 == 0 ? 32 : 16;
  const int64_t m_tiles = ceil_div(n_out > 0 ? n_out : 1, kCmM);
  // widest N tile (the gathered rows are staged once per N tile), halved while the launch would not cover the SMs once
  c.n_tile = c_out % 128 == 0 ? 128 : (c_out % 64 == 0 ? 64 : (c_out % 32 == 0 ? 32 : 16));
  while (c.n_tile > 32 && m_tiles * (c_out / c.n_tile) < kNumSMs) c.n_tile /= 2;
  // offset split of under-filled launches (deep, narrow levels: a few dozen row tiles, 27 offsets x C/KC chunks of strictly
  // sequential work each): the split that minimises  waves(ctas * ks) * (offsets per CTA + fixed prologue/epilogue) + cost of
  // summing ks partial tiles -- in particular never a split that spills a few CTAs into a second wave
  const int64_t ctas = m_tiles * (c_out / c.n_tile);
  const int smem = (kCmM + c.n_tile) * (c.kc * 2 + 16) * kCmStages + kCmMaxKV * kCmM * 4 + 128;
  int occ = (227 * 1024) / (smem + 1024);
  const int reg_occ = c.n_tile == 128 ? 2 : 3;   // accumulator registers: 128 fp32 per thread at NT = 128
  if (occ > reg_occ) occ = reg_occ;
  if (occ < 1) occ = 1;
  const int64_t slots = (int64_t)kNumSMs * occ;
  c.ksplit = 1;
  if (ctas < slots && kv > 1) {
    double best = 1e30;
    for (int ks = 1; ks <= 16 && ks <= kv; ++ks) {
      const double waves = (double)ceil_div(ctas * ks, slots);
      const double cost = waves * ((double)ceil_div(kv, ks) + 3.0) + 0.3 * ks;
      if (cost < best - 1e-9) { best = cost; c.ksplit = ks; }
    }
  }
  return c;
}

inline bool spconv_mma_supported(int dtype, int c_in, int c_out) {
  return (dtype == B2PC_F16 || dtype == B2PC_BF16) && c_in % 16 == 0 && c_out % 16 == 0;
}

// weight: [c_out][kv][c_in] (K-major: the KC channels of one output channel and offset are contiguous)
template <typename T, int KC, int NT>
__global__ void __launch_bounds__(128)
gather_gemm_mma_kernel(const T* __restrict__ feat, const T* __restrict__ weight, const T* __restrict__ bias,
                       const int32_t* __restrict__ pair, int64_t pair_stride, int64_t n_out, int c_in, int c_out, int kv, int flip,
                       T* __restrict__ out, int ksplit, float* __restrict__ acc) {
  using namespace mma;
  constexpr int S = kCmStages;
  constexpr int P = KC * 2 + 16;   // bytes per staged row
  constexpr int NTL = NT / 8;      // 8-column tiles per warp
  constexpr int STAGE = conv_mma_stage_bytes<KC, NT>();
  extern __shared__ __align__(128) uint8_t smem[];
  int32_t* idx_s = reinterpret_cast<int32_t*>(smem);                           // [kCmMaxKV][128]
  uint32_t* mask_s = reinterpret_cast<uint32_t*>(smem + kCmMaxKV * kCmM * 4);
  uint8_t* act_s = reinterpret_cast<uint8_t*>(mask_s + 1);                     // [kCmMaxKV]
  uint8_t* stage0 = smem + kCmMaxKV * kCmM * 4 + 128;
  const uint32_t stage0_u32 = smem_u32(stage0);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, tq = lane & 3;
  const int64_t row0 = (int64_t)blockIdx.x * kCmM;
  const int n0 = blockIdx.y * NT;
  const int n_cc = c_in / KC;

  float d[2][NTL][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < NTL; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) d[mt][nt][e] = 0.f;

  // kernel offsets are processed in chunks of kCmMaxKV (the rulebook slice of a chunk lives in shared memory)
  for (int kb = 0; kb < kv; kb += kCmMaxKV) {
    const int kcnt = min(kCmMaxKV, kv - kb);
    __syncthreads();   // the previous chunk's units are consumed by every warp
    if (tid == 0) *mask_s = 0;
    __syncthreads();
    {
      const int64_t j = row0 + tid;
      uint32_t wmask = 0;
      for (int k8 = 0; k8 < kcnt; k8 += 8) {
        int32_t v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {   // 8 independent loads in flight before the first use
          const int k = k8 + u;
          const int kp = flip ? kv - 1 - (kb + k) : kb + k;
          v[u] = (k < kcnt && j < n_out) ? __ldg(pair + (int64_t)kp * pair_stride + j) : -1;
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int k = k8 + u;
          if (k < kcnt) {
            idx_s[k * kCmM + tid] = v[u];
            if (__ballot_sync(0xFFFFFFFFu, v[u] >= 0)) wmask |= 1u << k;
          }
        }
      }
      if (lane == 0 && wmask) atomicOr(mask_s, wmask);
    }
    __syncthreads();
    uint32_t mask = *mask_s;
    if (ksplit > 1) {   // this CTA's share of the offsets: k % ksplit == blockIdx.z
      uint32_t mine = 0;
      for (int k = 0; k < kcnt; ++k)
        if ((kb + k) % ksplit == (int)blockIdx.z) mine |= 1u << k;
      mask &= mine;
    }
    const int n_act = __popc(mask);
    const int n_it = n_act * n_cc;   // unit = (active offset, channel chunk)
    if (tid < n_act) act_s[tid] = (uint8_t)__fns(mask, 0, tid + 1);   // active offsets of this chunk, in order
    __syncthreads();

    auto issue = [&](int it, int s) {
      const int a = it / n_cc, cc = it - a * n_cc;
      const int kl = act_s[a];
      const int c0 = cc * KC;
      const uint32_t st = stage0_u32 + s * STAGE;
      const int32_t src = idx_s[kl * kCmM + tid];
      const T* gp = feat + (int64_t)(src >= 0 ? src : 0) * c_in + c0;
#pragma unroll
      for (int p = 0; p < KC / 8; ++p) cp_async16(st + tid * P + p * 16, gp + p * 8, src >= 0);
      const T* wk = weight + ((int64_t)n0 * kv + kb + kl) * c_in + c0;
      constexpr int kPieces = NT * KC / 8;
#pragma unroll
      for (int q0 = 0; q0 < kPieces; q0 += kCmM) {
        const int q = q0 + tid;
        if (kPieces % kCmM == 0 || q < kPieces) {
          const int r = q / (KC / 8), pp = q % (KC / 8);
          cp_async16(st + kCmM * P + r * P + pp * 16, wk + (int64_t)r * kv * c_in + pp * 8, true);
        }
      }
    };
#pragma unroll
    for (int it = 0; it < S - 1; ++it) {
      if (it < n_it) issue(it, it);
      cp_async_commit();
    }
    for (int it = 0; it < n_it; ++it) {
      cp_async_wait<S - 2>();
      __syncthreads();   // unit `it` landed for every thread; every warp is done with unit it-1, whose stage unit it+S-1 reuses
      if (it + S - 1 < n_it) issue(it + S - 1, (it + S - 1) % S);
      cp_async_commit();
      const uint32_t a_st = stage0_u32 + (it % S) * STAGE, b_st = a_st + kCmM * P;
#pragma unroll
      for (int ks = 0; ks < KC / 16; ++ks) {
        uint32_t a[2][4];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt)
          ldsm_x4(a_st + (warp * 32 + mt * 16 + LdsmA::r(lane)) * P + (ks * 16 + LdsmA::c(lane)) * 2, a[mt]);
#pragma unroll
        for (int np = 0; np < NT / 16; ++np) {
          uint32_t b[4];
          ldsm_x4(b_st + (np * 16 + LdsmBnk::r(lane)) * P + (ks * 16 + LdsmBnk::c(lane)) * 2, b);
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            mma16816<T>(d[mt][2 * np], a[mt], b[0], b[1]);
            mma16816<T>(d[mt][2 * np + 1], a[mt], b[2], b[3]);
          }
        }
      }
    }
    cp_async_wait<0>();
  }
  // epilogue: thread (g, tq) holds rows g, g+8 of each 16-row tile, columns 2tq, 2tq+1 of each 8-column tile
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const int64_t j = row0 + warp * 32 + mt * 16 + g + r * 8;
      if (j >= n_out) continue;
#pragma unroll
      for (int nt = 0; nt < NTL; ++nt) {
        const int col = n0 + nt * 8 + 2 * tq;
        float v0 = d[mt][nt][2 * r], v1 = d[mt][nt][2 * r + 1];
        if (ksplit > 1) {   // this split's partial tile goes to its own slice (summed in a fixed order by conv_split_finish_kernel)
          *reinterpret_cast<float2*>(acc + ((int64_t)blockIdx.z * n_out + j) * c_out + col) = make_float2(v0, v1);
        } else {
          if (bias) { v0 += to_f32(bias[col]); v1 += to_f32(bias[col + 1]); }
          *reinterpret_cast<uint32_t*>(out + j * c_out + col) = pack2<T>(v0, v1);
        }
      }
    }
}

// out[j, c] = bias[c] + sum_z acc[z, j, c]   (offset-split path; fixed summation order)
template <typename T>
__global__ void __launch_bounds__(256)
conv_split_finish_kernel(const float* __restrict__ acc, int n_split, const T* __restrict__ bias, int64_t n_out, int c_out, T* __restrict__ out) {
  const int64_t total = n_out * c_out / 4;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    float4 v = reinterpret_cast<const float4*>(acc)[i];
    for (int z = 1; z < n_split; ++z) {
      const float4 w = reinterpret_cast<const float4*>(acc)[(int64_t)z * total + i];
      v.x += w.x; v.y += w.y; v.z += w.z; v.w += w.w;
    }
    const int c0 = (int)((i * 4) % c_out);
    float b0 = 0.f, b1 = 0.f, b2 = 0.f, b3 = 0.f;
    if (bias) { b0 = to_f32(bias[c0]); b1 = to_f32(bias[c0 + 1]); b2 = to_f32(bias[c0 + 2]); b3 = to_f32(bias[c0 + 3]); }
    reinterpret_cast<uint2*>(out)[i] = make_uint2(pack2<T>(v.x + b0, v.y + b1), pack2<T>(v.z + b2, v.w + b3));
  }
}

// wt[ci, k, co] = w[co, k, ci]: the backward-data pass as a forward pass over the transposed weights (K-major tiles)
template <typename T>
__global__ void __launch_bounds__(256)
conv_transpose_w_kernel(const T* __restrict__ w, int c_out, int kv, int c_in, T* __restrict__ wt) {
  __shared__ T tile[32][33];
  const int k = blockIdx.z, ci0 = blockIdx.x * 32, co0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int r = ty; r < 32; r += 8) {
    const int co = co0 + r, ci = ci0 + tx;
    if (co < c_out && ci < c_in) tile[r][tx] = w[((int64_t)co * kv + k) * c_in + ci];
  }
  __syncthreads();
  for (int r = ty; r < 32; r += 8) {
    const int ci = ci0 + r, co = co0 + tx;
    if (co < c_out && ci < c_in) wt[((int64_t)ci * kv + k) * c_out + co] = tile[tx][r];
  }
}

inline size_t conv_mma_split_bytes(const ConvMmaCfg& c, int64_t n_out, int c_out) {
  return c.ksplit > 1 ? align_up((size_t)c.ksplit * n_out * c_out * sizeof(float), 256) : 0;
}

// split partials (under-filled launches) + a transposed copy of the weights (backward-data calls)
inline size_t conv_mma_workspace_bytes(int64_t n_out, int c_in, int c_out, int kv) {
  if (c_in % 16 != 0 || c_out % 16 != 0) return 0;
  const ConvMmaCfg c = conv_mma_cfg(n_out, c_in, c_out, kv);
  return conv_mma_split_bytes(c, n_out, c_out) + align_up((size_t)kv * c_in * c_out * 2, 256) + 256;
}

template <typename T>
inline int launch_gather_gemm_mma_t(const void* feat, const void* weight, const void* bias, const int32_t* pair, int64_t pair_stride,
                                    int64_t n_out, int c_in, int c_out, int kv, int transpose_w, int flip, void* out, void* ws,
                                    cudaStream_t stream) {
  const ConvMmaCfg c = conv_mma_cfg(n_out, c_in, c_out, kv);
  float* acc = (float*)ws;
  const void* w = weight;
  if (transpose_w) {   // weight is [c_in(arg) rows = conv c_out][kv][c_out(arg)]: make the [c_out(arg)][kv][c_in(arg)] copy this pass reads
    T* wt = (T*)((char*)ws + conv_mma_split_bytes(c, n_out, c_out));
    dim3 tg((unsigned)ceil_div(c_out, 32), (unsigned)ceil_div(c_in, 32), (unsigned)kv);
    conv_transpose_w_kernel<T><<<tg, 256, 0, stream>>>((const T*)weight, c_in, kv, c_out, wt);
    count_launches(1);
    w = wt;
  }
  dim3 grid((unsigned)ceil_div(n_out, kCmM), c_out / c.n_tile, c.ksplit);
#define B2PC_CONV_LAUNCH(KC, NT)                                                                                                   \
  do {                                                                                                                             \
    constexpr int smem = conv_mma_smem_bytes<KC, NT>();                                                                            \
    cudaFuncSetAttribute(gather_gemm_mma_kernel<T, KC, NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);                   \
    gather_gemm_mma_kernel<T, KC, NT><<<grid, kCmM, smem, stream>>>((const T*)feat, (const T*)w, (const T*)bias, pair, pair_stride, \
                                                                    n_out, c_in, c_out, kv, flip, (T*)out, c.ksplit, acc);         \
  } while (0)
  if (c.kc == 32) {
    switch (c.n_tile) {
      case 128: B2PC_CONV_LAUNCH(32, 128); break;
      case 64: B2PC_CONV_LAUNCH(32, 64); break;
      case 32: B2PC_CONV_LAUNCH(32, 32); break;
      default: B2PC_CONV_LAUNCH(32, 16); break;
    }
  } else {
    switch (c.n_tile) {
      case 128: B2PC_CONV_LAUNCH(16, 128); break;
      case 64: B2PC_CONV_LAUNCH(16, 64); break;
      case 32: B2PC_CONV_LAUNCH(16, 32); break;
      default: B2PC_CONV_LAUNCH(16, 16); break;
    }
  }
#undef B2PC_CONV_LAUNCH
  count_launches(1);
  if (c.ksplit > 1) {
    int64_t fb = ceil_div(n_out * c_out / 4, 256);
    if (fb > kNumSMs * 8) fb = kNumSMs * 8;
    conv_split_finish_kernel<T><<<(int)fb, 256, 0, stream>>>(acc, c.ksplit, (const T*)bias, n_out, c_out, (T*)out);
    count_launches(1);
  }
  B2PC_CHECK_LAUNCH("spconv_gather_gemm(tensor core)");
  return B2PC_OK;
}

inline int launch_gather_gemm_mma(const void* feat, const void* weight, const void* bias, const int32_t* pair, int64_t pair_stride,
                                  int64_t n_out, int c_in, int c_out, int kv, int transpose_w, int flip, int dtype, void* out, void* ws,
                                  cudaStream_t stream) {
  if (n_out == 0) return B2PC_OK;
  if (dtype == B2PC_BF16)
    return launch_gather_gemm_mma_t<__nv_bfloat16>(feat, weight, bias, pair, pair_stride, n_out, c_in, c_out, kv, transpose_w, flip, out, ws, stream);
  return launch_gather_gemm_mma_t<__half>(feat, weight, bias, pair, pair_stride, n_out, c_in, c_out, kv, transpose_w, flip, out, ws, stream);
}

// ---------------------------------------------------------------------------------------------------------------------
// Weight gradient:   dW[co, k, ci] = sum_j dout[j, co] * feat[pair[k, j], ci]
// One CTA owns one kernel offset k, a BM tile of output channels and a BN tile of input channels, and sweeps its share of 64-row
// tiles of the rulebook (row tiles split % n_splits).  Per row tile the dout rows (A, read transposed by ldmatrix.trans: rows are
// the reduction axis) and the gathered feature rows (B, zero where the pair is absent) are staged through a 3-stage cp.async ring;
// warp w reduces rows 16w .. 16w+15 of every tile into its own BM x BN accumulator, and the four warp accumulators are summed in
// shared memory in a fixed order at the end.  Row-range splits are reduced afterwards in a fixed order (deterministic, no atomics).
constexpr int kWmRows = 64;     // rulebook rows per step (reduction chunk, 16 per warp)
constexpr int kWmStages = 3;

template <int BM, int BN> __host__ __device__ constexpr int wgrad_mma_stage_bytes() { return kWmRows * (BM * 2 + 16) + kWmRows * (BN * 2 + 16); }
template <int BM, int BN> __host__ __device__ constexpr int wgrad_mma_smem_bytes() {
  return kWmStages * wgrad_mma_stage_bytes<BM, BN>() > BM * BN * 4 ? kWmStages * wgrad_mma_stage_bytes<BM, BN>() : BM * BN * 4;
}

struct WgradMmaCfg { int bm, bn, n_splits; };

inline WgradMmaCfg wgrad_mma_cfg(int64_t n_out, int c_in, int c_out, int kv) {
  WgradMmaCfg c;
  c.bm = c_out % 64 == 0 ? 64 : (c_out % 32 == 0 ? 32 : 16);
  c.bn = c_in % 64 == 0 ? 64 : (c_in % 32 == 0 ? 32 : 16);
  const int64_t tiles = ceil_div(n_out > 0 ? n_out : 1, kWmRows);
  const int64_t ctas = (int64_t)kv * (c_out / c.bm) * (c_in / c.bn);
  int64_t sp = ceil_div((int64_t)4 * kNumSMs, ctas);   // about four CTAs per SM
  if (sp > tiles) sp = tiles;
  if (sp > 64) sp = 64;
  if (sp < 1) sp = 1;
  c.n_splits = (int)sp;
  return c;
}

inline bool wgrad_mma_supported(int dtype, int c_in, int c_out) {
  return (dtype == B2PC_F16 || dtype == B2PC_BF16) && c_in % 16 == 0 && c_out % 16 == 0;
}

inline size_t wgrad_mma_workspace_bytes(int64_t n_out, int c_in, int c_out, int kv) {
  if (c_in % 16 != 0 || c_out % 16 != 0) return 0;
  const WgradMmaCfg c = wgrad_mma_cfg(n_out, c_in, c_out, kv);
  return (size_t)c.n_splits * c_out * kv * c_in * sizeof(float) + 256;
}

template <typename T, int BM, int BN>
__global__ void __launch_bounds__(128)
bwd_weight_mma_kernel(const T* __restrict__ feat, const T* __restrict__ dout, const int32_t* __restrict__ pair, int64_t pair_stride,
                      int64_t n_out, int c_in, int c_out, int kv, int n_splits, float* __restrict__ partial) {
  using namespace mma;
  constexpr int S = kWmStages;
  constexpr int PA = BM * 2 + 16, PB = BN * 2 + 16;
  constexpr int MT = BM / 16, NTL = BN / 8;
  constexpr int STAGE = wgrad_mma_stage_bytes<BM, BN>();
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t smem0 = smem_u32(smem);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, tq = lane & 3;
  int bx = blockIdx.x;
  const int n_nt = c_in / BN, n_mt = c_out / BM;
  const int nt_i = bx % n_nt; bx /= n_nt;
  const int mt_i = bx % n_mt; bx /= n_mt;
  const int k = bx;
  const int split = blockIdx.y;
  const int co0 = mt_i * BM, ci0 = nt_i * BN;
  const int64_t n_tiles = ceil_div(n_out, kWmRows);
  const int my_tiles = split < n_tiles ? (int)ceil_div(n_tiles - split, n_splits) : 0;
  const int32_t* pk = pair + (int64_t)k * pair_stride;

  float d[MT][NTL][4];
#pragma unroll
  for (int mt = 0; mt < MT; ++mt)
#pragma unroll
    for (int nt = 0; nt < NTL; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) d[mt][nt][e] = 0.f;

  auto issue = [&](int it, int s) {
    const int64_t r0 = (int64_t)(split + (int64_t)it * n_splits) * kWmRows;
    const uint32_t a_st = smem0 + s * STAGE, b_st = a_st + kWmRows * PA;
#pragma unroll
    for (int q0 = 0; q0 < kWmRows * BM / 8; q0 += 128) {
      const int q = q0 + tid;
      if ((kWmRows * BM / 8) % 128 == 0 || q < kWmRows * BM / 8) {
        const int r = q / (BM / 8), p = q % (BM / 8);
        const int64_t j = r0 + r;
        cp_async16(a_st + r * PA + p * 16, dout + (j < n_out ? j : 0) * c_out + co0 + p * 8, j < n_out);
      }
    }
#pragma unroll
    for (int q0 = 0; q0 < kWmRows * BN / 8; q0 += 128) {
      const int q = q0 + tid;
      if ((kWmRows * BN / 8) % 128 == 0 || q < kWmRows * BN / 8) {
        const int r = q / (BN / 8), p = q % (BN / 8);
        const int64_t j = r0 + r;
        const int32_t src = j < n_out ? __ldg(pk + j) : -1;
        cp_async16(b_st + r * PB + p * 16, feat + (int64_t)(src >= 0 ? src : 0) * c_in + ci0 + p * 8, src >= 0);
      }
    }
  };
#pragma unroll
  for (int it = 0; it < S - 1; ++it) {
    if (it < my_tiles) issue(it, it);
    cp_async_commit();
  }
  for (int it = 0; it < my_tiles; ++it) {
    cp_async_wait<S - 2>();
    __syncthreads();
    if (it + S - 1 < my_tiles) issue(it + S - 1, (it + S - 1) % S);
    cp_async_commit();
    const uint32_t a_st = smem0 + (it % S) * STAGE, b_st = a_st + kWmRows * PA;
    uint32_t a[MT][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
      ldsm_x4_t(a_st + (warp * 16 + LdsmAkm::r(lane)) * PA + (mt * 16 + LdsmAkm::c(lane)) * 2, a[mt]);
#pragma unroll
    for (int np = 0; np < BN / 16; ++np) {
      uint32_t b[4];
      ldsm_x4_t(b_st + (warp * 16 + LdsmBkn::r(lane)) * PB + (np * 16 + LdsmBkn::c(lane)) * 2, b);
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        mma16816<T>(d[mt][2 * np], a[mt], b[0], b[1]);
        mma16816<T>(d[mt][2 * np + 1], a[mt], b[2], b[3]);
      }
    }
  }
  cp_async_wait<0>();
  // sum of the four warp accumulators in shared memory, warp 0 first (fixed order), then partial[split][co][k][ci]
  float* red = reinterpret_cast<float*>(smem);
  for (int w = 0; w < 4; ++w) {
    __syncthreads();
    if (warp == w) {
#pragma unroll
      for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int nt = 0; nt < NTL; ++nt)
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int row = mt * 16 + g + (e >> 1) * 8, col = nt * 8 + 2 * tq + (e & 1);
            red[row * BN + col] = w == 0 ? d[mt][nt][e] : red[row * BN + col] + d[mt][nt][e];
          }
    }
  }
  __syncthreads();
  for (int q = tid; q < BM * BN; q += 128) {
    const int row = q / BN, col = q % BN;
    partial[(((int64_t)split * c_out + co0 + row) * kv + k) * c_in + ci0 + col] = red[q];
  }
}

template <typename T>
inline int launch_bwd_weight_mma_t(const void* feat, const void* dout, const int32_t* pair, int64_t pair_stride, int64_t n_out,
                                   int c_in, int c_out, int kv, float* dweight, void* ws, cudaStream_t stream) {
  const WgradMmaCfg c = wgrad_mma_cfg(n_out, c_in, c_out, kv);
  dim3 grid((unsigned)(kv * (c_out / c.bm) * (c_in / c.bn)), (unsigned)c.n_splits);
#define B2PC_WGRAD_LAUNCH(BM, BN)                                                                                                  \
  do {                                                                                                                             \
    constexpr int smem = wgrad_mma_smem_bytes<BM, BN>();                                                                           \
    cudaFuncSetAttribute(bwd_weight_mma_kernel<T, BM, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);                    \
    bwd_weight_mma_kernel<T, BM, BN><<<grid, 128, smem, stream>>>((const T*)feat, (const T*)dout, pair, pair_stride, n_out, c_in,  \
                                                                  c_out, kv, c.n_splits, (float*)ws);                              \
  } while (0)
#define B2PC_WGRAD_BN(BM)                            \
  do {                                               \
    if (c.bn == 64) B2PC_WGRAD_LAUNCH(BM, 64);       \
    else if (c.bn == 32) B2PC_WGRAD_LAUNCH(BM, 32);  \
    else B2PC_WGRAD_LAUNCH(BM, 16);                  \
  } while (0)
  if (c.bm == 64) B2PC_WGRAD_BN(64);
  else if (c.bm == 32) B2PC_WGRAD_BN(32);
  else B2PC_WGRAD_BN(16);
#undef B2PC_WGRAD_BN
#undef B2PC_WGRAD_LAUNCH
  const int64_t elems = (int64_t)c_out * kv * c_in;
  int rb = (int)ceil_div(elems, 256);
  if (rb > kNumSMs * 8) rb = kNumSMs * 8;
  reduce_splits_kernel<<<rb, 256, 0, stream>>>((const float*)ws, elems, c.n_splits, dweight);
  count_launches(2);
  B2PC_CHECK_LAUNCH("spconv_bwd_weight(tensor core)");
  return B2PC_OK;
}

inline int launch_bwd_weight_mma(const void* feat, const void* dout, const int32_t* pair, int64_t pair_stride, int64_t n_out, int c_in,
                                 int c_out, int kv, int dtype, float* dweight, void* ws, cudaStream_t stream) {
  if (dtype == B2PC_BF16)
    return launch_bwd_weight_mma_t<__nv_bfloat16>(feat, dout, pair, pair_stride, n_out, c_in, c_out, kv, dweight, ws, stream);
  return launch_bwd_weight_mma_t<__half>(feat, dout, pair, pair_stride, n_out, c_in, c_out, kv, dweight, ws, stream);
}

}  // namespace b2pc
