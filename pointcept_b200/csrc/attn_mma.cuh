// Patch attention on the Hopper tensor cores (mma.sync m16n8k16, fp32 accumulators in registers), head_dim 16.
//
// Forward: one CTA = one (sequence, head, 64-query tile); four warps, warp w owns query rows 16w .. 16w+15 for the whole sweep, so
// the softmax state (row max, row sum, output row) never leaves the registers of the quad that holds the row.  Per block of 64 keys:
//     S  = Q K_j^T      8 MMAs (N = 8 keys each, K = 16 = head_dim), Q fragment loaded once, K_j by ldmatrix
//     P  = exp2(c*S - m) in registers; the accumulator layout of two 8-key tiles is the A fragment of one 16-key step
//     O  = O*corr + P V_j   4 x 2 MMAs, V_j by ldmatrix.trans (V stays [key][channel] in shared memory)
// K / V blocks stream through a 3-stage cp.async ring.  D = 16 makes this kernel exp-bound (64 MMA flops per exp), not tensor-bound;
// its shared memory (14 KB) lets many CTAs share an SM so that loads, MMAs and exponentials of different tiles overlap.
#pragma once
#include "attn_simt.cuh"   // kLog2e, kLn2
#include "common.cuh"
#include "mma.cuh"

namespace b2pc {

constexpr int kAmQ = 64;       // queries per CTA (16 per warp)
constexpr int kAmN = 64;       // keys per block
constexpr int kAmStages = 3;   // K/V ring depth

// GATHER = true (serialized attention, ptv3m1:188,216 fused in): qkv holds POINT rows [N, 3, H, 16]; slot t of the padded patch
// sequence reads point row gidx[t] (= order[pad][t]) and writes its output to point row sidx[t] when sidx[t] >= 0 (the slot is
// the point's primary slot; borrowed filler slots have sidx < 0 and are dropped) -- the [order] gather and the [inverse]
// gather of the reference happen inside the tile loads / the epilogue and the padded qkv / out tensors never exist.
// Rows past the end of a ragged sequence are zero-filled by the loads (never read from the next sequence) and their
// probabilities are set to zero, so non-finite values in neighbouring sequences cannot leak in.
template <typename T, bool GATHER>
__global__ void __launch_bounds__(128)
attn_fwd_mma_kernel(const T* __restrict__ qkv, const int32_t* __restrict__ cu, int64_t t_total, int H, float scale,
                    T* __restrict__ out, float* __restrict__ lse, const int32_t* __restrict__ gidx, const int32_t* __restrict__ sidx) {
  using namespace mma;
  constexpr int D = 16;
  __shared__ __align__(128) uint8_t q_s[kAmQ * 32];
  __shared__ __align__(128) uint8_t kv_s[kAmStages][2][kAmN * 32];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, tq = lane & 3;
  const int seq = blockIdx.y, h = blockIdx.z;
  const int64_t s0 = cu[seq];
  const int len = (int)(cu[seq + 1] - s0);
  const int q0 = blockIdx.x * kAmQ;
  if (q0 >= len) return;
  const int nblk = (len + kAmN - 1) / kAmN;
  const int64_t row_stride = (int64_t)3 * H * D;   // elements between consecutive tokens
  const int64_t row_base = GATHER ? 0 : s0;        // GATHER: rows are addressed through gidx
  const T* base_q = qkv + row_base * row_stride + h * D;
  const T* base_k = base_q + H * D;
  const int32_t* gix = GATHER ? gidx + s0 : nullptr;
  const int lr = tid >> 1, lh = tid & 1;           // loading thread -> (tile row, 16-byte half)
  {
    const bool ok = q0 + lr < len;
    const int64_t prow = ok ? (GATHER ? (int64_t)__ldg(gix + q0 + lr) : (int64_t)(q0 + lr)) : 0;
    cp_async16(smem_u32(q_s) + row32_off(lr, lh), base_q + prow * row_stride + lh * 8, ok);
  }
  auto load_kv = [&](int blk, int stage) {
    const int k0 = blk * kAmN;
    const bool ok = k0 + lr < len;
    const int64_t prow = ok ? (GATHER ? (int64_t)__ldg(gix + k0 + lr) : (int64_t)(k0 + lr)) : 0;
    const T* src = base_k + prow * row_stride + lh * 8;
    cp_async16(smem_u32(kv_s[stage][0]) + row32_off(lr, lh), src, ok);
    cp_async16(smem_u32(kv_s[stage][1]) + row32_off(lr, lh), src + H * D, ok);
  };
  load_kv(0, 0);
  cp_async_commit();
  if (nblk > 1) load_kv(1, 1);
  cp_async_commit();

  const float c = scale * kLog2e;
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};   // rows g, g+8 of the warp's 16
  float o[2][4];
#pragma unroll
  for (int nt = 0; nt < 2; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) o[nt][e] = 0.f;
  uint32_t qa[4];

  for (int j = 0; j < nblk; ++j) {
    const int stage = j % kAmStages;
    cp_async_wait<1>();
    __syncthreads();   // block j landed for every thread; every warp is done with block j-1, whose stage block j+2 reuses
    if (j == 0) ldsm_x4(smem_u32(q_s) + row32_off(warp * 16 + LdsmA::r(lane), LdsmA::c(lane) >> 3), qa);
    if (j + 2 < nblk) load_kv(j + 2, (j + 2) % kAmStages);
    cp_async_commit();
    const uint32_t ks = smem_u32(kv_s[stage][0]), vs = smem_u32(kv_s[stage][1]);
    float s[8][4];
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      uint32_t b[4];
      ldsm_x4(ks + row32_off(np * 16 + LdsmBnk::r(lane), LdsmBnk::c(lane) >> 3), b);
#pragma unroll
      for (int e = 0; e < 4; ++e) { s[2 * np][e] = 0.f; s[2 * np + 1][e] = 0.f; }
      mma16816<T>(s[2 * np], qa, b[0], b[1]);
      mma16816<T>(s[2 * np + 1], qa, b[2], b[3]);
    }
    const int nvalid = len - j * kAmN;
    if (nvalid < kAmN) {
#pragma unroll
      for (int nt = 0; nt < 8; ++nt)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (nt * 8 + 2 * tq + (e & 1) >= nvalid) s[nt][e] = -INFINITY;
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      mx[0] = fmaxf(mx[0], fmaxf(s[nt][0], s[nt][1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[nt][2], s[nt][3]));
    }
    float corr[2], mn[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xFFFFFFFFu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xFFFFFFFFu, mx[r], 2));
      mn[r] = fmaxf(m[r], mx[r] * c);   // every block holds at least one valid key: finite
      corr[r] = ex2(m[r] - mn[r]);
      l[r] *= corr[r];
      m[r] = mn[r];
    }
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) { o[nt][0] *= corr[0]; o[nt][1] *= corr[0]; o[nt][2] *= corr[1]; o[nt][3] *= corr[1]; }
    uint32_t pa[4][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float p0 = ex2(fmaf(s[nt][0], c, -mn[0])), p1 = ex2(fmaf(s[nt][1], c, -mn[0]));
      const float p2 = ex2(fmaf(s[nt][2], c, -mn[1])), p3 = ex2(fmaf(s[nt][3], c, -mn[1]));
      l[0] += p0 + p1;
      l[1] += p2 + p3;
      pa[nt >> 1][(nt & 1) * 2] = pack2<T>(p0, p1);
      pa[nt >> 1][(nt & 1) * 2 + 1] = pack2<T>(p2, p3);
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t b[4];
      ldsm_x4_t(vs + row32_off(kk * 16 + LdsmBkn::r(lane), LdsmBkn::c(lane) >> 3), b);
      mma16816<T>(o[0], pa[kk], b[0], b[1]);
      mma16816<T>(o[1], pa[kk], b[2], b[3]);
    }
  }
  cp_async_wait<0>();
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xFFFFFFFFu, l[r], 1);
    l[r] += __shfl_xor_sync(0xFFFFFFFFu, l[r], 2);
    const int qi = q0 + warp * 16 + g + r * 8;
    if (qi >= len) continue;
    const float inv = 1.f / l[r];
    const int64_t orow = GATHER ? (int64_t)__ldg(sidx + s0 + qi) : s0 + qi;
    if (orow >= 0) {
      T* dst = out + (orow * H + h) * D + 2 * tq;
      *reinterpret_cast<uint32_t*>(dst) = pack2<T>(o[0][2 * r] * inv, o[0][2 * r + 1] * inv);
      *reinterpret_cast<uint32_t*>(dst + 8) = pack2<T>(o[1][2 * r] * inv, o[1][2 * r + 1] * inv);
    }
    if (tq == 0) lse[(int64_t)h * t_total + s0 + qi] = (m[r] + log2f(l[r])) * kLn2;
  }
}

inline bool attn_mma_supported(int dtype, int head_dim) {
  return head_dim == 16 && (dtype == B2PC_F16 || dtype == B2PC_BF16);
}

// gidx / sidx non-null: serialized (gather-fused) mode, see the kernel comment
inline int launch_attn_fwd_mma(const void* qkv, int dtype, const int32_t* cu, int n_seq, int max_seqlen, int64_t t, int H, int D,
                               float scale, void* out, float* lse, cudaStream_t stream, const int32_t* gidx = nullptr,
                               const int32_t* sidx = nullptr) {
  (void)D;
  if (n_seq == 0 || t == 0) return B2PC_OK;
  dim3 grid((unsigned)ceil_div(max_seqlen, kAmQ), n_seq, H);
#define B2PC_ATTN_FWD_LAUNCH(T)                                                                                                  \
  do {                                                                                                                           \
    if (gidx) attn_fwd_mma_kernel<T, true><<<grid, 128, 0, stream>>>((const T*)qkv, cu, t, H, scale, (T*)out, lse, gidx, sidx);     \
    else attn_fwd_mma_kernel<T, false><<<grid, 128, 0, stream>>>((const T*)qkv, cu, t, H, scale, (T*)out, lse, nullptr, nullptr);   \
  } while (0)
  if (dtype == B2PC_BF16) B2PC_ATTN_FWD_LAUNCH(__nv_bfloat16);
  else B2PC_ATTN_FWD_LAUNCH(__half);
#undef B2PC_ATTN_FWD_LAUNCH
  count_launches(1);
  B2PC_CHECK_LAUNCH("patch_attn_fwd(tensor core)");
  return B2PC_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
// Backward, in two deterministic kernels: every gradient element is formed by one thread in a fixed order and written once (no
// atomics), so the same inputs give the same bits on every run.
// dK / dV: one CTA = one (sequence, head, block of 64 keys); warp w owns key rows 16w .. 16w+15 and sweeps the queries in blocks
// of 64, everything in the transposed frame so that the CTA-owned dK / dV accumulate in registers across the sweep:
//     S^T  = K_j Q_i^T,  dP^T = V_j dO_i^T        M = 16 keys per warp, N = 64 queries, K = 16
//     P^T  = exp2(c S^T - lse2_i),  dS^T = P^T * (dP^T - delta_i)   (registers; the accumulators are the A fragments below)
//     dV_j += P^T dO_i,  dK_j += dS^T Q_i         M = 16 keys, N = 16, K = 64 queries (dO_i / Q_i by ldmatrix.trans)
// dQ: one CTA = one (sequence, head, block of 64 queries), the frame of the forward kernel: warp w owns query rows 16w .. 16w+15
// and sweeps the key blocks in order, recomputing S and dP (dQ_i = sum_j dS_ij K_j, K = 64 keys per step).
constexpr int kAbK = 64;        // keys per CTA
constexpr int kAbQ = 64;        // queries per sweep step
constexpr int kAbStages = 3;    // Q / dO ring depth
constexpr int kAbStageBytes = kAbQ * 32 * 2 + kAbQ * 4 * 2;   // Q | dO | -lse*log2(e) | -delta

// GATHER = true: serialized mode (see the forward kernel): qkv / dout / dqkv hold POINT rows; slot t reads point row gidx[t],
// its dO is dout[sidx[t]] when sidx[t] >= 0 and zero otherwise (the output of a borrowed filler slot was dropped); dK / dV of a
// primary slot go straight to the point's row of dqkv, those of filler slot with sidx = -(r+1) to row r of `side` [n_dup, 2, H, 16]
// (added to the point's row afterwards: a point owns at most one filler slot besides its primary one).
template <typename T, bool GATHER>
__global__ void __launch_bounds__(128)
attn_bwd_mma_kernel(const T* __restrict__ dout, const T* __restrict__ qkv, const float* __restrict__ nlse2,
                    const float* __restrict__ ndelta, const int32_t* __restrict__ cu, int64_t t_total, int H, float scale,
                    T* __restrict__ dqkv, const int32_t* __restrict__ gidx, const int32_t* __restrict__ sidx, T* __restrict__ side) {
  using namespace mma;
  constexpr int D = 16;
  __shared__ __align__(128) uint8_t k_s[kAbK * 32];
  __shared__ __align__(128) uint8_t v_s[kAbK * 32];
  __shared__ __align__(128) uint8_t st_s[kAbStages][kAbStageBytes];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, tq = lane & 3;
  const int seq = blockIdx.y, h = blockIdx.z;
  const int64_t s0 = cu[seq];
  const int len = (int)(cu[seq + 1] - s0);
  const int k0 = blockIdx.x * kAbK;
  if (k0 >= len) return;
  const int nblk = (len + kAbQ - 1) / kAbQ;
  const int64_t row_stride = (int64_t)3 * H * D;
  const int64_t row_base = GATHER ? 0 : s0;
  const T* base_q = qkv + row_base * row_stride + h * D;
  const T* base_k = base_q + H * D;
  const T* base_do = dout + row_base * H * D + h * D;
  const int32_t* gix = GATHER ? gidx + s0 : nullptr;
  const int32_t* six = GATHER ? sidx + s0 : nullptr;
  const float* base_lse = nlse2 + (int64_t)h * t_total + s0;
  const float* base_dl = ndelta + (int64_t)h * t_total + s0;
  const int lr = tid >> 1, lh = tid & 1;   // loading thread -> (tile row, 16-byte half)
  {
    const bool ok = k0 + lr < len;
    const int64_t prow = ok ? (GATHER ? (int64_t)__ldg(gix + k0 + lr) : (int64_t)(k0 + lr)) : 0;
    const T* src = base_k + prow * row_stride + lh * 8;
    cp_async16(smem_u32(k_s) + row32_off(lr, lh), src, ok);
    cp_async16(smem_u32(v_s) + row32_off(lr, lh), src + H * D, ok);
  }
  auto load_q = [&](int blk, int stage) {
    uint8_t* st = st_s[stage];
    const int q = blk * kAbQ + lr;
    const bool ok = q < len;
    const int64_t qrow = ok ? (GATHER ? (int64_t)__ldg(gix + q) : (int64_t)q) : 0;
    const int64_t drow = ok ? (GATHER ? (int64_t)__ldg(six + q) : (int64_t)q) : -1;
    cp_async16(smem_u32(st) + row32_off(lr, lh), base_q + qrow * row_stride + lh * 8, ok);
    cp_async16(smem_u32(st + kAbQ * 32) + row32_off(lr, lh), base_do + (drow >= 0 ? drow : 0) * (H * D) + lh * 8, drow >= 0);
    // -lse*log2(e) (threads 0-63) and -delta (threads 64-127) of the 64 queries; zero where the query does not exist
    const int r = tid & 63, q2 = blk * kAbQ + r;
    const float* src = (tid < 64 ? base_lse : base_dl) + q2;
    cp_async4(smem_u32(st + kAbQ * 64 + (tid >> 6) * (kAbQ * 4) + r * 4), q2 < len ? src : base_lse, q2 < len);
  };
  load_q(0, 0);
  cp_async_commit();
  if (nblk > 1) load_q(1, 1);
  cp_async_commit();

  const float c = scale * kLog2e;
  float dv[2][4], dk[2][4];
#pragma unroll
  for (int nt = 0; nt < 2; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) { dv[nt][e] = 0.f; dk[nt][e] = 0.f; }
  uint32_t ka[4], va[4];

  for (int i = 0; i < nblk; ++i) {
    uint8_t* st = st_s[i % kAbStages];
    cp_async_wait<1>();
    __syncthreads();   // block i landed; every warp is done with block i-1, whose stage block i+2 reuses
    if (i == 0) {
      ldsm_x4(smem_u32(k_s) + row32_off(warp * 16 + LdsmA::r(lane), LdsmA::c(lane) >> 3), ka);
      ldsm_x4(smem_u32(v_s) + row32_off(warp * 16 + LdsmA::r(lane), LdsmA::c(lane) >> 3), va);
    }
    if (i + 2 < nblk) load_q(i + 2, (i + 2) % kAbStages);
    cp_async_commit();
    const uint32_t qs = smem_u32(st), dos = smem_u32(st + kAbQ * 32);
    float s[8][4], dp[8][4];
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      uint32_t bq[4], bd[4];
      ldsm_x4(qs + row32_off(np * 16 + LdsmBnk::r(lane), LdsmBnk::c(lane) >> 3), bq);
      ldsm_x4(dos + row32_off(np * 16 + LdsmBnk::r(lane), LdsmBnk::c(lane) >> 3), bd);
#pragma unroll
      for (int e = 0; e < 4; ++e) { s[2 * np][e] = 0.f; s[2 * np + 1][e] = 0.f; dp[2 * np][e] = 0.f; dp[2 * np + 1][e] = 0.f; }
      mma16816<T>(s[2 * np], ka, bq[0], bq[1]);
      mma16816<T>(s[2 * np + 1], ka, bq[2], bq[3]);
      mma16816<T>(dp[2 * np], va, bd[0], bd[1]);
      mma16816<T>(dp[2 * np + 1], va, bd[2], bd[3]);
    }
    const float* lse_s = reinterpret_cast<const float*>(st + kAbQ * 64);
    const float* dl_s = lse_s + kAbQ;
    uint32_t pa[4][4], da[4][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float2 l2 = *reinterpret_cast<const float2*>(lse_s + nt * 8 + 2 * tq);
      const float2 d2 = *reinterpret_cast<const float2*>(dl_s + nt * 8 + 2 * tq);
      const float p0 = ex2(fmaf(s[nt][0], c, l2.x)), p1 = ex2(fmaf(s[nt][1], c, l2.y));
      const float p2 = ex2(fmaf(s[nt][2], c, l2.x)), p3 = ex2(fmaf(s[nt][3], c, l2.y));
      const float e0 = p0 * (dp[nt][0] + d2.x), e1 = p1 * (dp[nt][1] + d2.y);
      const float e2 = p2 * (dp[nt][2] + d2.x), e3 = p3 * (dp[nt][3] + d2.y);
      pa[nt >> 1][(nt & 1) * 2] = pack2<T>(p0, p1);
      pa[nt >> 1][(nt & 1) * 2 + 1] = pack2<T>(p2, p3);
      da[nt >> 1][(nt & 1) * 2] = pack2<T>(e0, e1);
      da[nt >> 1][(nt & 1) * 2 + 1] = pack2<T>(e2, e3);
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t bd[4], bq[4];
      ldsm_x4_t(dos + row32_off(kk * 16 + LdsmBkn::r(lane), LdsmBkn::c(lane) >> 3), bd);
      ldsm_x4_t(qs + row32_off(kk * 16 + LdsmBkn::r(lane), LdsmBkn::c(lane) >> 3), bq);
      mma16816<T>(dv[0], pa[kk], bd[0], bd[1]);
      mma16816<T>(dv[1], pa[kk], bd[2], bd[3]);
      mma16816<T>(dk[0], da[kk], bq[0], bq[1]);
      mma16816<T>(dk[1], da[kk], bq[2], bq[3]);
    }
  }
  cp_async_wait<0>();
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int ki = k0 + warp * 16 + g + r * 8;
    if (ki >= len) continue;
    T *dkp, *dvp;
    if (GATHER) {
      const int64_t si = __ldg(six + ki);
      if (si >= 0) {
        dkp = dqkv + ((si * 3 + 1) * H + h) * D;
        dvp = dqkv + ((si * 3 + 2) * H + h) * D;
      } else {
        dkp = side + (((-si - 1) * 2 + 0) * H + h) * D;
        dvp = side + (((-si - 1) * 2 + 1) * H + h) * D;
      }
    } else {
      dkp = dqkv + (((s0 + ki) * 3 + 1) * H + h) * D;
      dvp = dqkv + (((s0 + ki) * 3 + 2) * H + h) * D;
    }
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      *reinterpret_cast<uint32_t*>(dkp + nt * 8 + 2 * tq) = pack2<T>(dk[nt][2 * r] * scale, dk[nt][2 * r + 1] * scale);
      *reinterpret_cast<uint32_t*>(dvp + nt * 8 + 2 * tq) = pack2<T>(dv[nt][2 * r], dv[nt][2 * r + 1]);
    }
  }
}

// dQ (see above).  Q / dO rows, -lse*log2(e) and -delta of the CTA's 64 queries are loaded once, K / V blocks stream through the
// ring of the forward kernel.  dS is rounded to the operand type before the dQ MMA, as in the dK kernel.  Serialized mode: slot t
// writes row sidx[t] of dqkv; a filler slot (sidx < 0) has dO = 0 and delta = 0, hence dQ = 0, and writes nothing.
template <typename T, bool GATHER>
__global__ void __launch_bounds__(128)
attn_bwd_dq_mma_kernel(const T* __restrict__ dout, const T* __restrict__ qkv, const float* __restrict__ nlse2,
                       const float* __restrict__ ndelta, const int32_t* __restrict__ cu, int64_t t_total, int H, float scale,
                       T* __restrict__ dqkv, const int32_t* __restrict__ gidx, const int32_t* __restrict__ sidx) {
  using namespace mma;
  constexpr int D = 16;
  __shared__ __align__(128) uint8_t q_s[kAmQ * 32];
  __shared__ __align__(128) uint8_t do_s[kAmQ * 32];
  __shared__ __align__(128) uint8_t kv_s[kAmStages][2][kAmN * 32];

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, tq = lane & 3;
  const int seq = blockIdx.y, h = blockIdx.z;
  const int64_t s0 = cu[seq];
  const int len = (int)(cu[seq + 1] - s0);
  const int q0 = blockIdx.x * kAmQ;
  if (q0 >= len) return;
  const int nblk = (len + kAmN - 1) / kAmN;
  const int64_t row_stride = (int64_t)3 * H * D;
  const int64_t row_base = GATHER ? 0 : s0;
  const T* base_q = qkv + row_base * row_stride + h * D;
  const T* base_k = base_q + H * D;
  const T* base_do = dout + row_base * H * D + h * D;
  const int32_t* gix = GATHER ? gidx + s0 : nullptr;
  const int32_t* six = GATHER ? sidx + s0 : nullptr;
  const int lr = tid >> 1, lh = tid & 1;   // loading thread -> (tile row, 16-byte half)
  {
    const bool ok = q0 + lr < len;
    const int64_t qrow = ok ? (GATHER ? (int64_t)__ldg(gix + q0 + lr) : (int64_t)(q0 + lr)) : 0;
    const int64_t drow = ok ? (GATHER ? (int64_t)__ldg(six + q0 + lr) : (int64_t)(q0 + lr)) : -1;
    cp_async16(smem_u32(q_s) + row32_off(lr, lh), base_q + qrow * row_stride + lh * 8, ok);
    cp_async16(smem_u32(do_s) + row32_off(lr, lh), base_do + (drow >= 0 ? drow : 0) * (H * D) + lh * 8, drow >= 0);
  }
  auto load_kv = [&](int blk, int stage) {
    const int k0 = blk * kAmN;
    const bool ok = k0 + lr < len;
    const int64_t prow = ok ? (GATHER ? (int64_t)__ldg(gix + k0 + lr) : (int64_t)(k0 + lr)) : 0;
    const T* src = base_k + prow * row_stride + lh * 8;
    cp_async16(smem_u32(kv_s[stage][0]) + row32_off(lr, lh), src, ok);
    cp_async16(smem_u32(kv_s[stage][1]) + row32_off(lr, lh), src + H * D, ok);
  };
  load_kv(0, 0);
  cp_async_commit();
  if (nblk > 1) load_kv(1, 1);
  cp_async_commit();

  // -lse*log2(e) and -delta of the thread's two query rows (zero for rows past the sequence end, which are not written)
  float nl[2], nd[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int qi = q0 + warp * 16 + g + r * 8;
    const bool ok = qi < len;
    nl[r] = ok ? __ldg(nlse2 + (int64_t)h * t_total + s0 + qi) : 0.f;
    nd[r] = ok ? __ldg(ndelta + (int64_t)h * t_total + s0 + qi) : 0.f;
  }
  const float c = scale * kLog2e;
  float dq[2][4];
#pragma unroll
  for (int nt = 0; nt < 2; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) dq[nt][e] = 0.f;
  uint32_t qa[4], doa[4];

  for (int j = 0; j < nblk; ++j) {
    const int stage = j % kAmStages;
    cp_async_wait<1>();
    __syncthreads();   // block j landed for every thread; every warp is done with block j-1, whose stage block j+2 reuses
    if (j == 0) {
      ldsm_x4(smem_u32(q_s) + row32_off(warp * 16 + LdsmA::r(lane), LdsmA::c(lane) >> 3), qa);
      ldsm_x4(smem_u32(do_s) + row32_off(warp * 16 + LdsmA::r(lane), LdsmA::c(lane) >> 3), doa);
    }
    if (j + 2 < nblk) load_kv(j + 2, (j + 2) % kAmStages);
    cp_async_commit();
    const uint32_t ks = smem_u32(kv_s[stage][0]), vs = smem_u32(kv_s[stage][1]);
    float s[8][4], dp[8][4];
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      uint32_t bk[4], bv[4];
      ldsm_x4(ks + row32_off(np * 16 + LdsmBnk::r(lane), LdsmBnk::c(lane) >> 3), bk);
      ldsm_x4(vs + row32_off(np * 16 + LdsmBnk::r(lane), LdsmBnk::c(lane) >> 3), bv);
#pragma unroll
      for (int e = 0; e < 4; ++e) { s[2 * np][e] = 0.f; s[2 * np + 1][e] = 0.f; dp[2 * np][e] = 0.f; dp[2 * np + 1][e] = 0.f; }
      mma16816<T>(s[2 * np], qa, bk[0], bk[1]);
      mma16816<T>(s[2 * np + 1], qa, bk[2], bk[3]);
      mma16816<T>(dp[2 * np], doa, bv[0], bv[1]);
      mma16816<T>(dp[2 * np + 1], doa, bv[2], bv[3]);
    }
    const int nvalid = len - j * kAmN;
    uint32_t da[4][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      float e[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float p = (nt * 8 + 2 * tq + (i & 1) < nvalid) ? ex2(fmaf(s[nt][i], c, nl[i >> 1])) : 0.f;
        e[i] = p * (dp[nt][i] + nd[i >> 1]);
      }
      da[nt >> 1][(nt & 1) * 2] = pack2<T>(e[0], e[1]);
      da[nt >> 1][(nt & 1) * 2 + 1] = pack2<T>(e[2], e[3]);
    }
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      uint32_t b[4];
      ldsm_x4_t(ks + row32_off(kk * 16 + LdsmBkn::r(lane), LdsmBkn::c(lane) >> 3), b);
      mma16816<T>(dq[0], da[kk], b[0], b[1]);
      mma16816<T>(dq[1], da[kk], b[2], b[3]);
    }
  }
  cp_async_wait<0>();
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int qi = q0 + warp * 16 + g + r * 8;
    if (qi >= len) continue;
    const int64_t orow = GATHER ? (int64_t)__ldg(six + qi) : s0 + qi;
    if (orow < 0) continue;
    T* dst = dqkv + ((orow * 3 + 0) * H + h) * D + 2 * tq;
    *reinterpret_cast<uint32_t*>(dst) = pack2<T>(dq[0][2 * r] * scale, dq[0][2 * r + 1] * scale);
    *reinterpret_cast<uint32_t*>(dst + 8) = pack2<T>(dq[1][2 * r] * scale, dq[1][2 * r + 1] * scale);
  }
}

// serialized mode: dqkv[dup_point[r], 1 + which, h, :] += side[r, which, h, :]   (one thread per (r, which, h), 16 channels)
template <typename T>
__global__ void __launch_bounds__(256)
attn_dup_add_kernel(const T* __restrict__ side, const int32_t* __restrict__ dup_point, int64_t n_dup, int H, T* __restrict__ dqkv) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;   // over n_dup * 2 * H
  if (i >= n_dup * 2 * H) return;
  const int h = (int)(i % H);
  const int which = (int)((i / H) % 2);
  const int64_t r = i / (2 * H);
  const T* src = side + i * 16;
  T* dst = dqkv + (((int64_t)dup_point[r] * 3 + 1 + which) * H + h) * 16;
#pragma unroll
  for (int e = 0; e < 16; ++e) dst[e] = from_f32<T>(to_f32(dst[e]) + to_f32(src[e]));
}

inline size_t attn_bwd_mma_workspace_bytes(int64_t t, int H, int D, int64_t n_dup = 0) {
  (void)D;
  return 2 * align_up((size_t)t * H * sizeof(float), 256) + align_up((size_t)n_dup * 2 * H * 16 * 2, 256) + 256;
}

// ndelta[h, t] = -sum_d dout*out,  nlse2[h, t] = -lse[h, t] * log2(e)   (the signs / scale the main kernel's FMAs want);
// serialized mode: dout / out are point rows, slot t uses row sidx[t] and gets delta = 0 when it is a filler slot
template <typename T>
__global__ void __launch_bounds__(256)
attn_bwd_prep_kernel(const T* __restrict__ dout, const T* __restrict__ out, const float* __restrict__ lse, int64_t t_total, int H,
                     float* __restrict__ ndelta, float* __restrict__ nlse2, const int32_t* __restrict__ sidx) {
  const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;  // over T*H, (t, h) order
  if (i >= t_total * H) return;
  const int64_t t = i / H;
  const int h = (int)(i % H);
  float acc = 0.f;
  const int64_t row = sidx ? (int64_t)sidx[t] : t;
  if (row >= 0) {
    const uint4* a = reinterpret_cast<const uint4*>(dout + (row * H + h) * 16);
    const uint4* b = reinterpret_cast<const uint4*>(out + (row * H + h) * 16);
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const uint4 va = a[q], vb = b[q];
      const uint32_t wa[4] = {va.x, va.y, va.z, va.w}, wb[4] = {vb.x, vb.y, vb.z, vb.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const T* pa = reinterpret_cast<const T*>(&wa[e]);
        const T* pb = reinterpret_cast<const T*>(&wb[e]);
        acc = fmaf(to_f32(pa[0]), to_f32(pb[0]), acc);
        acc = fmaf(to_f32(pa[1]), to_f32(pb[1]), acc);
      }
    }
  }
  ndelta[(int64_t)h * t_total + t] = -acc;
  nlse2[(int64_t)h * t_total + t] = -lse[(int64_t)h * t_total + t] * kLog2e;
}

// gidx non-null: serialized mode (dout / qkv / out / dqkv are point rows; see the kernel comments)
template <typename T>
inline int launch_attn_bwd_mma_t(const void* dout, const void* qkv, const void* out, const float* lse, const int32_t* cu, int n_seq,
                                 int max_seqlen, int64_t t, int H, float scale, void* dqkv, void* ws, cudaStream_t stream,
                                 const int32_t* gidx, const int32_t* sidx, const int32_t* dup_point, int64_t n_dup) {
  float* delta = (float*)ws;                                                        // holds -delta
  float* nlse2 = (float*)((char*)ws + align_up((size_t)t * H * sizeof(float), 256));  // holds -lse * log2(e)
  T* side = (T*)((char*)ws + 2 * align_up((size_t)t * H * sizeof(float), 256));
  attn_bwd_prep_kernel<T><<<(unsigned)ceil_div(t * H, 256), 256, 0, stream>>>((const T*)dout, (const T*)out, lse, t, H, delta, nlse2, sidx);
  dim3 grid((unsigned)ceil_div(max_seqlen, kAbK), n_seq, H);
  dim3 grid_dq((unsigned)ceil_div(max_seqlen, kAmQ), n_seq, H);
  if (gidx) {
    attn_bwd_mma_kernel<T, true><<<grid, 128, 0, stream>>>((const T*)dout, (const T*)qkv, nlse2, delta, cu, t, H, scale, (T*)dqkv, gidx,
                                                          sidx, side);
    attn_bwd_dq_mma_kernel<T, true><<<grid_dq, 128, 0, stream>>>((const T*)dout, (const T*)qkv, nlse2, delta, cu, t, H, scale, (T*)dqkv,
                                                                gidx, sidx);
  } else {
    attn_bwd_mma_kernel<T, false><<<grid, 128, 0, stream>>>((const T*)dout, (const T*)qkv, nlse2, delta, cu, t, H, scale, (T*)dqkv,
                                                           nullptr, nullptr, nullptr);
    attn_bwd_dq_mma_kernel<T, false><<<grid_dq, 128, 0, stream>>>((const T*)dout, (const T*)qkv, nlse2, delta, cu, t, H, scale, (T*)dqkv,
                                                                 nullptr, nullptr);
  }
  count_launches(3);
  if (gidx && n_dup > 0) {
    attn_dup_add_kernel<T><<<(unsigned)ceil_div(n_dup * 2 * H, 256), 256, 0, stream>>>(side, dup_point, n_dup, H, (T*)dqkv);
    count_launches(1);
  }
  B2PC_CHECK_LAUNCH("patch_attn_bwd(tensor core)");
  return B2PC_OK;
}

inline int launch_attn_bwd_mma(const void* dout, const void* qkv, const void* out, const float* lse, int dtype, const int32_t* cu,
                               int n_seq, int max_seqlen, int64_t t, int H, int D, float scale, void* dqkv, void* ws,
                               cudaStream_t stream, const int32_t* gidx = nullptr, const int32_t* sidx = nullptr,
                               const int32_t* dup_point = nullptr, int64_t n_dup = 0) {
  (void)D;
  if (n_seq == 0 || t == 0) return B2PC_OK;
  if (dtype == B2PC_F16)
    return launch_attn_bwd_mma_t<__half>(dout, qkv, out, lse, cu, n_seq, max_seqlen, t, H, scale, dqkv, ws, stream, gidx, sidx, dup_point, n_dup);
  return launch_attn_bwd_mma_t<__nv_bfloat16>(dout, qkv, out, lse, cu, n_seq, max_seqlen, t, H, scale, dqkv, ws, stream, gidx, sidx, dup_point,
                                              n_dup);
}

}  // namespace b2pc
