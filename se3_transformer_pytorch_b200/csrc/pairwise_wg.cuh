// The fused pairwise kernel on the Hopper tensor cores, shared by the direct path (pairwise_tc.cu: A = the radial-trunk
// output g, K = 128, bias from the weight image) and the low-rank path (pairwise_lr.cu: A = the radial coordinates U,
// K = Kp <= 64, bias folded into the GEMM):
//
//   R[e, n] = sum_k A[e, k] W[n, k] (+ b[n]),     n = if_local * 32 + o_local
//   out[e, o, p] (+)= sum_{i,f} R[e, (i,f,o)] * T[e, i, f, p]
//
// One CTA = (tile of 128 edges) x (block of 32 output channels), looping over ceil(Ci*F/4) steps of 4 (i,f) pairs.
// fp32 parity with a 3-pass fp16 split: A = A_hi + A_lo, W = W_hi + W_lo, R ~= A_hi W_hi + A_lo W_hi + A_hi W_lo.
//
// 384 threads.  Warp 0 streams the W units (32 KiB: [hi 128 x 64 | lo 128 x 64] fp16, SW128) and the T stages (plus the
// bias of the direct path) with TMA bulk copies into mbarrier rings; warpgroups 1 and 2 own 64 edge rows each.  At start they
// split their rows of A into fp16 hi / lo images in shared memory (SW128, stationary for the whole CTA); per step and per
// half of the 128 columns, each issues a chain of m64n64k16 wgmma (both operands from shared memory) into 32 fp32
// registers and contracts them with T straight from the accumulator fragment, keeping out[2 rows, 8 channels, P] in
// registers across the whole step loop.  The two warpgroups interleave, so one's MMAs overlap the other's contraction.
#pragma once
#include "common.cuh"
#include "tc_ptx.cuh"

namespace se3 {

constexpr int kPwThreads = 384;
constexpr uint32_t kPwUnitBytes = 2 * kSubBytes;   // one W unit: [hi 16 KiB | lo 16 KiB]
constexpr uint32_t kPwBiasBytes = 512;              // 128 fp32 (direct path)
constexpr int kPwTStages = 3;

struct PwParams {
  const float* A;          // [E, lda] fp32
  const uint8_t* w_img;
  const float* T;          // [edge tiles][steps][4 (i,f)][PH][128 edges][4] fp32
  float* out;
  float* dumpR;            // direct path, tests only: R + bias of step 0, [edge tiles, Co/32, 128 edges, 128 columns]
  int64_t E;
  int lda, NIFB, n_mt, n_ob, accumulate;
  int nk16, spu, NU;       // low-rank path: K16 blocks per step, steps per W unit, W units per channel block
  int64_t out_es;          // floats between consecutive edges of the output
  int out_os;              // floats between consecutive output channels of an edge
  int p_off[7];            // position of component p inside an output row
};

// TC: direct path (K = 128: two W units per step, [hi|lo] of k-half 0 then 1, followed by the bias; A sub-tiles = 2);
// otherwise the low-rank path (one W unit holds spu steps side by side along K; A sub-tiles = 1).
template <int P, bool TC, bool kDumpR, int WS>
__global__ void __launch_bounds__(kPwThreads, 1)
pairwise_wg_kernel(const PwParams prm) {
  constexpr int PH = (P + 3) / 4;
  constexpr uint32_t kTBytes = PH * 8192u;              // 4 (i,f) x PH x 128 edges x 16 B
  constexpr uint32_t kTStageBytes = kTBytes + (TC ? kPwBiasBytes : 0u);
  constexpr int NSUB = TC ? 2 : 1;                      // 64-wide K sub-tiles of A
  constexpr uint32_t kABytes = 2u * NSUB * kSubBytes;   // [hi sub-tiles | lo sub-tiles]
  constexpr uint32_t kTileBytes = 2u * kPwUnitBytes + kPwBiasBytes;   // direct path: one step of the image
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* base_ptr = smem_raw + (base - raw);
  const uint32_t sA = base;
  const uint32_t sW = sA + kABytes;                     // + slot * kPwUnitBytes
  const uint32_t sT = sW + WS * kPwUnitBytes;           // + stage * kTStageBytes (bias after the T block)
  const uint32_t sBar = sT + kPwTStages * kTStageBytes;
  const uint32_t bar_w_full = sBar;
  const uint32_t bar_w_empty = bar_w_full + 8 * WS;
  const uint32_t bar_t_full = bar_w_empty + 8 * WS;
  const uint32_t bar_t_empty = bar_t_full + 8 * kPwTStages;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int NIFB = prm.NIFB;
  const int ob = (int)(blockIdx.x % prm.n_ob);
  const int64_t mt = blockIdx.x / prm.n_ob;

  if (threadIdx.x == 0) {
    for (int s = 0; s < WS; ++s) {
      mbar_init(bar_w_full + 8 * s, 1);
      mbar_init(bar_w_empty + 8 * s, 8);       // one arrival per consumer warp
    }
    for (int s = 0; s < kPwTStages; ++s) {
      mbar_init(bar_t_full + 8 * s, 1);
      mbar_init(bar_t_empty + 8 * s, 8);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0 && lane == 0) {
      // ===================== producer: W units and T stages, in step order =====================
      const uint8_t* tsrc = reinterpret_cast<const uint8_t*>(prm.T) + (size_t)mt * NIFB * kTBytes;
      int u = 0;                                 // next W unit to load
      for (int s = 0; s < NIFB; ++s) {
        const int u_end = TC ? 2 * (s + 1) : (s / prm.spu + 1);
        for (; u < u_end; ++u) {
          const int slot = u % WS;
          mbar_wait(bar_w_empty + 8 * slot, ((uint32_t)(u / WS) & 1u) ^ 1u);
          mbar_arrive_expect_tx(bar_w_full + 8 * slot, kPwUnitBytes);
          const uint8_t* src = TC ? prm.w_img + ((size_t)ob * NIFB + (u >> 1)) * kTileBytes + (u & 1) * kPwUnitBytes
                                  : prm.w_img + ((size_t)ob * prm.NU + u) * kPwUnitBytes;
          bulk_g2s(sW + slot * kPwUnitBytes, src, kPwUnitBytes, bar_w_full + 8 * slot);
        }
        const int ts = s % kPwTStages;
        mbar_wait(bar_t_empty + 8 * ts, ((uint32_t)(s / kPwTStages) & 1u) ^ 1u);
        mbar_arrive_expect_tx(bar_t_full + 8 * ts, kTStageBytes);
        bulk_g2s(sT + ts * kTStageBytes, tsrc + (size_t)s * kTBytes, kTBytes, bar_t_full + 8 * ts);
        if (TC)
          bulk_g2s(sT + ts * kTStageBytes + kTBytes, prm.w_img + ((size_t)ob * NIFB + s) * kTileBytes + 2 * kPwUnitBytes, kPwBiasBytes,
                   bar_t_full + 8 * ts);
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
    const int ct = threadIdx.x - 128;            // 0..255
    const int wg = ct >> 7;                      // consumer warpgroup: edge rows [64 wg, 64 wg + 64)
    const int w4 = (ct >> 5) & 3;
    // ---- A operand: rows of A (fp32) -> fp16 hi / lo images, SW128 K-major; two threads per row, 64 * NSUB / 2 columns each
    {
      const int r = ct >> 1, k0 = (ct & 1) * 32 * NSUB;
      const int64_t eg = mt * SE3_TILE_E + r;
      const bool live = eg < prm.E;
      const float* arow = prm.A + (size_t)(live ? eg : 0) * prm.lda;
#pragma unroll
      for (int c = 0; c < 4 * NSUB; ++c) {       // 8 k values = one 16-byte chunk per iteration
        const int k = k0 + c * 8;
        float4 x0 = live ? __ldg(reinterpret_cast<const float4*>(arow + k)) : make_float4(0.f, 0.f, 0.f, 0.f);
        float4 x1 = live ? __ldg(reinterpret_cast<const float4*>(arow + k + 4)) : make_float4(0.f, 0.f, 0.f, 0.f);
        uint4 hi, lo;
        split_h2(x0.x, x0.y, hi.x, lo.x);
        split_h2(x0.z, x0.w, hi.y, lo.y);
        split_h2(x1.x, x1.y, hi.z, lo.z);
        split_h2(x1.z, x1.w, hi.w, lo.w);
        const uint32_t off = sw128_off(r, k);
        *reinterpret_cast<uint4*>(base_ptr + off) = hi;
        *reinterpret_cast<uint4*>(base_ptr + NSUB * kSubBytes + off) = lo;
      }
      fence_proxy_async();
      consumer_sync();
    }

    // this thread's rows of the accumulator fragment: r0 = 16 w4 + lane/4 (+8) inside the warpgroup's 64 rows
    const int el0 = wg * 64 + w4 * 16 + (lane >> 2);
    const float4* Tsm = reinterpret_cast<const float4*>(base_ptr + (sT - base));
    float acc[2][8][P];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int b = 0; b < 8; ++b)
#pragma unroll
        for (int p = 0; p < P; ++p) acc[a][b][p] = 0.f;

    const int nk = TC ? 8 : prm.nk16;
    for (int s = 0; s < NIFB; ++s) {
      const int sub = TC ? 0 : s % prm.spu;
      const int u0 = TC ? 2 * s : s / prm.spu;
      mbar_wait(bar_w_full + 8 * (u0 % WS), (uint32_t)(u0 / WS) & 1u);
      if (TC) mbar_wait(bar_w_full + 8 * ((u0 + 1) % WS), (uint32_t)((u0 + 1) / WS) & 1u);
      const int ts = s % kPwTStages;
      bool t_ready = false;
#pragma unroll
      for (int h = 0; h < 2; ++h) {              // columns [64 h, 64 h + 64): (i,f) slots 2h, 2h+1
        float R[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) R[i] = 0.f;
        wgmma_fence();
#pragma unroll
        for (int pass = 0; pass < 3; ++pass) {   // A_hi W_hi, A_lo W_hi, A_hi W_lo
#pragma unroll
          for (int j = 0; j < (TC ? 8 : 4); ++j) {
            if (j >= nk) break;
            const int u = TC ? u0 + (j >> 2) : u0;
            const uint32_t kofs = TC ? (uint32_t)(j & 3) * 32u : (uint32_t)(sub * nk + j) * 32u;
            const uint32_t a = sA + (pass == 1 ? NSUB * kSubBytes : 0u) + (uint32_t)(j >> 2) * kSubBytes + wg * 8192u + (uint32_t)(j & 3) * 32u;
            const uint32_t b = sW + (uint32_t)(u % WS) * kPwUnitBytes + (pass == 2 ? kSubBytes : 0u) + h * 8192u + kofs;
            wgmma_ss_n64(R, wg_desc_sw128(a), wg_desc_sw128(b), (pass | j) != 0);
          }
        }
        wgmma_commit();
        wgmma_wait0();
        if (h == 1) {
          // every MMA of this step has read its W units: release the ones no later step uses
          const bool last_of_unit = TC || sub == prm.spu - 1 || s == NIFB - 1;
          __syncwarp();
          if (last_of_unit && lane == 0) {
            mbar_arrive(bar_w_empty + 8 * (u0 % WS));
            if (TC) mbar_arrive(bar_w_empty + 8 * ((u0 + 1) % WS));
          }
        }
        if (!t_ready) {
          mbar_wait(bar_t_full + 8 * ts, (uint32_t)(s / kPwTStages) & 1u);
          t_ready = true;
        }
        const float* bias = reinterpret_cast<const float*>(base_ptr + (sT - base) + ts * kTStageBytes + kTBytes);
#pragma unroll
        for (int hs = 0; hs < 2; ++hs) {         // (i,f) slot ifl = 2h + hs: fragment registers [16 hs, 16 hs + 16)
          const int ifl = 2 * h + hs;
          float tv[2][PH * 4];
#pragma unroll
          for (int rs = 0; rs < 2; ++rs)
#pragma unroll
            for (int h4 = 0; h4 < PH; ++h4) {
              const float4 t4 = Tsm[(size_t)ts * (kTStageBytes / 16) + (ifl * PH + h4) * 128 + el0 + 8 * rs];
              tv[rs][h4 * 4 + 0] = t4.x; tv[rs][h4 * 4 + 1] = t4.y; tv[rs][h4 * 4 + 2] = t4.z; tv[rs][h4 * 4 + 3] = t4.w;
            }
#pragma unroll
          for (int ii = 0; ii < 16; ++ii) {
            const int i = 16 * hs + ii;
            const int rs = (ii >> 1) & 1;
            const int oi = ((ii >> 2) << 1) | (ii & 1);              // channel o_local = 8 (ii/4) + 2 (lane%4) + ii%2
            const int ol = 8 * (ii >> 2) + 2 * (lane & 3) + (ii & 1);
            float rv = R[i];
            if (TC) rv += bias[ifl * 32 + ol];
            if (kDumpR && s == 0 && mt < prm.n_mt)
              prm.dumpR[(((size_t)mt * prm.n_ob + ob) * 128 + el0 + 8 * rs) * 128 + ifl * 32 + ol] = rv;
#pragma unroll
            for (int p = 0; p < P; ++p) acc[rs][oi][p] = fmaf(rv, tv[rs][p], acc[rs][oi][p]);
          }
        }
      }
      // T / bias stage fully consumed
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_t_empty + 8 * ts);
    }
    // write out[e, ob*32 + o_local, p] (+ what is there)
#pragma unroll
    for (int rs = 0; rs < 2; ++rs) {
      const int64_t e = mt * SE3_TILE_E + el0 + 8 * rs;
      if (e < prm.E) {
#pragma unroll
        for (int oi = 0; oi < 8; ++oi) {
          const int o = ob * SE3_TILE_O + 8 * (oi >> 1) + 2 * (lane & 3) + (oi & 1);
          float* dst = prm.out + (size_t)e * prm.out_es + (size_t)o * prm.out_os;
          float prev[P];
#pragma unroll
          for (int p = 0; p < P; ++p) prev[p] = prm.accumulate ? __ldcg(dst + prm.p_off[p]) : 0.f;
#pragma unroll
          for (int p = 0; p < P; ++p) dst[prm.p_off[p]] = acc[rs][oi][p] + prev[p];
        }
      }
    }
  }
}

template <int P, bool TC, int WS>
static constexpr size_t pw_smem_bytes() {
  constexpr int PH = (P + 3) / 4;
  return 1024 + 2u * (TC ? 2 : 1) * kSubBytes + WS * kPwUnitBytes + kPwTStages * (PH * 8192u + (TC ? kPwBiasBytes : 0u)) + 256;
}

template <int P, bool TC, bool kDumpR, int WS>
static int launch_pw(const PwParams& prm, cudaStream_t s) {
  constexpr size_t smem = pw_smem_bytes<P, TC, WS>();
  static_assert(smem <= 227 * 1024, "shared memory of one CTA");
  auto kern = pairwise_wg_kernel<P, TC, kDumpR, WS>;
  SE3_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<(unsigned)((int64_t)prm.n_mt * prm.n_ob), kPwThreads, smem, s>>>(prm);
  SE3_LAUNCH_OK();
  return SE3_OK;
}

}  // namespace se3
