// K4z: the fused pairwise kernel of the production path (low-rank radial basis + edge-aligned frames, DESIGN.md 4.5) as ONE
// tensor-core GEMM per (degree_out, |m|) with the A operand generated on the fly.
//
// In the edge-aligned frame (DESIGN.md 4.4) the output component m of degree lo of one ConvSE3 is
//     m = 0 :  out'[e,o]   = sum_{li} sum_i  w0[e,o,i]  x'_li[e,i,0]
//     m > 0 :  out'[e,o,+] = sum_{li>=m} sum_i  a[e,o,i] x'[e,i,+m] - b[e,o,i] x'[e,i,-m]
//              out'[e,o,-] = sum_{li>=m} sum_i  b[e,o,i] x'[e,i,+m] + a[e,o,i] x'[e,i,-m]
// (reference S:237-254, 326-343 re-associated), and every radial weight is a short dot product with the per-edge radial
// coordinates U of its degree pair, w[e,o,i] = sum_k U[e,k] F'[(o,i),k] (DESIGN.md 4.2; K = r+1 <= 16 per sub-segment).
// Instead of forming w the sums are exchanged:
//     out'[e,o,c] = sum_{(li,i,f,k)}  Z_c[e,(li,i,f,k)] * F'[o,(li,i,f,k)],        Z_c[e,(li,i,f,k)] = +-U_li[e,k] x'_li[e,i,+-m]
// one GEMM with M = edges, N = output channels, K = sum_li C_in * F * 16, whose A operand Z is an outer product per edge:
// it costs E*C_in*16 multiplies to make (C_out times fewer than there are radial weights) and is produced by the CUDA cores
// straight into the A-operand registers of wgmma, split z = hi + lo in fp16 for the 3-pass fp32-parity MMA
// (hi*hi + lo*hi + hi*lo).  Nothing per radial weight ever touches the SIMT pipe.
//
// MODE 3 evaluates the |m| > 0 case with three real products per complex one (Gauss): with c = x'[+m], d = x'[-m],
//     S1 = sum (a+b) c,   S2 = sum a (d-c),   S3 = sum b (c+d);    out'[+] = S1 - S3,   out'[-] = S1 + S2
// i.e. three accumulators, each fed by its own weight set (a+b, a, b) and its own Z: 3 instead of 4 K = 16 GEMM units per
// (edge, o, i).  Chunk c of stage s belongs to weight set (4 s + c) % 3; the drain combines them.
//
// CTA = 128 edges x NC channels (a slice of an N-wide tile of the weight image; MODE 1 / 4: NC = 128, one accumulator;
// MODE 2: NC = 64, components (+m, -m) in two accumulators fed by the same B tiles; MODE 3: NC = 64, three accumulators).
// 384 threads: warp 0 streams the weight image (TMA bulk copies into an mbarrier ring); warpgroups 1 and 2 own 64 edge rows
// each, generate Z for their rows, issue m64 x NC x 16 wgmma with A from registers and B from shared memory, and keep the
// fp32 partial sums: tensor-core accumulation truncates, so every `flush_stages` stages the accumulators are added into
// registers with round-to-nearest adds and restarted.  MODE 1 / 3 commit one wgmma group per K chunk and generate the next chunk
// while the previous chunks' MMAs are in flight, with X loaded into registers a stage (MODE 1) or a 3-stage period (MODE 3)
// ahead; MODE 2 / 4 wait for their MMAs every stage.
#include "common.cuh"
#include "tc_ptx.cuh"
#include <algorithm>
#include <cstdlib>
#include <type_traits>

namespace se3 {

constexpr int kZThreads = 384;
constexpr int kZMaxSeg = 16;
constexpr uint32_t kZWRingBytes = 196608;     // shared memory for the weight ring

template <int V>
using ic = std::integral_constant<int, V>;

// f(ic<0>()), ..., f(ic<N - 1>()): fully unrolled, the index a compile-time constant in every call
template <class F, int... I>
__device__ __forceinline__ void static_for_seq(F&& f, std::integer_sequence<int, I...>) {
  (f(ic<I>()), ...);
}
template <int N, class F>
__device__ __forceinline__ void static_for(F&& f) {
  static_for_seq(f, std::make_integer_sequence<int, N>());
}

struct ZSeg {
  const float* U;      // [E, 64] fp32 (this sub-segment reads columns 0..15 from the pointer given)
  const float* X;      // rotated neighbour features [tiles][Ci][ncomp][128]
  int Ci, ncomp, cplus, cminus, n_stage, pad;
};

struct ZParams {
  ZSeg seg[kZMaxSeg];
  int n_seg;
  const uint8_t* w_img;      // [n_nt][S][hi: N x 128 B | lo: N x 128 B], SW128 K-major, 64 K values (4 chunks) per stage
  const float* sx;           // [E] power-of-two scale of the edge's neighbour features (keeps Z inside the fp16 range)
  float* out;
  int64_t E;
  int64_t out_es;            // floats per edge row of out
  int comp_off[2];           // offset of the component plane(s) inside an edge row
  int n_mt, n_nt, S, flush_stages;
};

// A fragment of one K = 16 chunk for rows (r0, r0 + 8), columns (kq, kq+1, kq+8, kq+9): v[row][4] -> fp16 hi / lo pairs
__device__ __forceinline__ void z_frag(const float (&v)[2][4], uint32_t (&hi)[4], uint32_t (&lo)[4]) {
  split_h2(v[0][0], v[0][1], hi[0], lo[0]);
  split_h2(v[1][0], v[1][1], hi[1], lo[1]);
  split_h2(v[0][2], v[0][3], hi[2], lo[2]);
  split_h2(v[1][2], v[1][3], hi[3], lo[3]);
}

template <int NR>
__device__ __forceinline__ void z_mma3(float (&d)[NR], const uint32_t (&hi)[4], const uint32_t (&lo)[4], uint64_t b_hi, uint64_t b_lo,
                                       uint32_t scale_d = 1) {
  if constexpr (NR == 64) {
    wgmma_rs_n128(d, hi, b_hi, scale_d);
    wgmma_rs_n128(d, lo, b_hi);
    wgmma_rs_n128(d, hi, b_lo);
  } else {
    wgmma_rs_n64(d, hi, b_hi, scale_d);
    wgmma_rs_n64(d, lo, b_hi);
    wgmma_rs_n64(d, hi, b_lo);
  }
}

template <int MODE, int N, int NC>
__global__ void __launch_bounds__(kZThreads, 1)
zgemm_kernel(const __grid_constant__ ZParams prm) {
  static_assert((MODE == 1 || MODE == 4) ? NC == 128 : NC == 64, "CTA width");
  static_assert(N % NC == 0 && (MODE == 1 || N == 128), "weight image tile");
  constexpr int NA = (MODE == 3) ? 3 : (MODE == 2) ? 2 : 1;   // accumulators
  constexpr int NO = (MODE == 2 || MODE == 3) ? 2 : 1;        // output planes
  constexpr int NR = NC / 2;                                   // fragment registers of one m64 x NC fp32 accumulator
  constexpr int NH = N / NC;                                   // CTAs per tile of the weight image
  constexpr uint32_t kImgStage = 2u * N * 128u;                // one stage of the weight image: [hi N rows | lo N rows] x 128 B
  constexpr uint32_t kStageBytes = 2u * NC * 128u;             // what one CTA keeps of it: its NC rows of hi and of lo
  constexpr int WS = (kZWRingBytes / kStageBytes > 8) ? 8 : (int)(kZWRingBytes / kStageBytes);

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t sW = base;
  const uint32_t bar_w_full = sW + WS * kStageBytes;
  const uint32_t bar_w_empty = bar_w_full + 8 * WS;

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
  const int S = prm.S, FS = prm.flush_stages;
  const int n_ct = prm.n_nt * NH;
  const int ctile = (int)(blockIdx.x % n_ct);
  const int64_t mt = blockIdx.x / n_ct;
  const int nt = ctile / NH, hs = ctile % NH;

  if (threadIdx.x == 0) {
    for (int s = 0; s < WS; ++s) {
      mbar_init(bar_w_full + 8 * s, 1);
      mbar_init(bar_w_empty + 8 * s, 8);       // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0 && lane == 0) {
      // ===================== weight producer =====================
      const uint8_t* wsrc = prm.w_img + (size_t)nt * S * kImgStage + (size_t)hs * NC * 128u;
      for (int s = 0; s < S; ++s) {
        const int slot = s % WS;
        mbar_wait(bar_w_empty + 8 * slot, ((uint32_t)(s / WS) & 1u) ^ 1u);
        mbar_arrive_expect_tx(bar_w_full + 8 * slot, kStageBytes);
        bulk_g2s(sW + slot * kStageBytes, wsrc + (size_t)s * kImgStage, NC * 128u, bar_w_full + 8 * slot);
        bulk_g2s(sW + slot * kStageBytes + NC * 128u, wsrc + (size_t)s * kImgStage + N * 128u, NC * 128u, bar_w_full + 8 * slot);
      }
    }
    return;
  }
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  // ===================== Z generators + MMA + fp32 partial sums =====================
  const int ct = threadIdx.x - 128;
  const int r0 = (ct >> 7) * 64 + ((ct >> 5) & 3) * 16 + (lane >> 2);    // rows r0, r0 + 8 of the edge tile
  const int kq = 2 * (lane & 3);                                         // columns kq, kq+1, kq+8, kq+9 of every K chunk
  int64_t eg[2];
  bool live[2];
  float sxe[2];
#pragma unroll
  for (int rs = 0; rs < 2; ++rs) {
    eg[rs] = mt * SE3_TILE_E + r0 + 8 * rs;
    live[rs] = eg[rs] < prm.E;
    sxe[rs] = (live[rs] && MODE != 4) ? prm.sx[eg[rs]] : 1.f;
  }
  float D[NA][NR], acc[NO][NR];
#pragma unroll
  for (int a = 0; a < NA; ++a)
#pragma unroll
    for (int j = 0; j < NR; ++j) D[a][j] = 0.f;
#pragma unroll
  for (int a = 0; a < NO; ++a)
#pragma unroll
    for (int j = 0; j < NR; ++j) acc[a][j] = 0.f;
  int blk_start = 0;
  // MODE 1 / 3 restart a drained accumulator with the first MMA that writes it (scale-d = 0) instead of zeroing its registers,
  // so D is written only by wgmma (bit a: accumulator a is drained).  Every stage writes every accumulator, so each block of
  // flush_stages stages restarts all of them before the next drain.
  int fresh = 0;

  auto release = [&](int s) {                  // every MMA that read the weight slot of stage s has retired
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_w_empty + 8 * (s % WS));
  };
  // the accumulators are added into the fp32 partial sums at the end of each block of flush_stages stages, and after the last
  auto drain_after = [&](int s) { return s + 1 == S || s + 1 - blk_start == FS; };
  auto drain = [&](int s) {
#pragma unroll
    for (int j = 0; j < NR; ++j) {
      if (MODE == 3) {
        acc[0][j] += D[0][j] - D[NA - 1][j];
        acc[1][j] += D[0][j] + D[NA > 1 ? 1 : 0][j];
      } else {
#pragma unroll
        for (int a = 0; a < NA; ++a) acc[a][j] += D[a][j];
      }
      if (MODE == 2 || MODE == 4)
#pragma unroll
        for (int a = 0; a < NA; ++a) D[a][j] = 0.f;
    }
    fresh = (1 << NA) - 1;
    blk_start = s + 1;
  };
  // MODE 2 / 4: the MMAs of stage s retire before the next stage is generated
  auto finish_stage = [&](int s) {
    wgmma_commit();
    wgmma_wait0();
    release(s);
    if (drain_after(s)) drain(s);
  };

  // MODE 1 / 3: one commit group per K chunk, so the MMAs of the last ZR - 1 chunks stay in flight while the next chunk's A
  // fragments are generated
  constexpr int ZR = (MODE == 3) ? 2 : 4;
  float u[2][4];                               // U[e, kq, kq+1, kq+8, kq+9] * sx[e] of rows r0, r0 + 8 (current segment)
  auto zf = [&](const float (&y)[2], uint32_t (&hi)[4], uint32_t (&lo)[4]) {
    float v[2][4];
#pragma unroll
    for (int rs = 0; rs < 2; ++rs)
#pragma unroll
      for (int q = 0; q < 4; ++q) v[rs][q] = u[rs][q] * y[rs];
    z_frag(v, hi, lo);
  };
  // chunk C of stage s into accumulator A.  The wait retires chunk k - ZR, whose A fragment registers the new chunk reuses; at
  // C == ZR - 1 that is the last chunk of stage s - 1, so its weight slot goes back.
  auto chunk_mma = [&](auto cc, auto ac, int s, const float (&y)[2], uint64_t b_hi, uint64_t b_lo) {
    constexpr int C = decltype(cc)::value, A = decltype(ac)::value;
    wgmma_wait<ZR - 1>();
    if (C == ZR - 1 && s != blk_start) release(s - 1);     // stage s - 1 was not drained: its slot is still held
    uint32_t hi[4], lo[4];
    zf(y, hi, lo);
    wgmma_fence();
    z_mma3<NR>(D[A], hi, lo, b_hi + 2 * C, b_lo + 2 * C, ((fresh >> A) & 1) ^ 1);
    fresh &= ~(1 << A);
    wgmma_commit();
  };
  auto end_stage = [&](int s) {
    if (drain_after(s)) {
      wgmma_wait0();
      release(s);
      drain(s);
    }
  };
  auto wait_stage = [&](int s, uint64_t& b_hi, uint64_t& b_lo) {
    mbar_wait(bar_w_full + 8 * (s % WS), (uint32_t)(s / WS) & 1u);
    const uint32_t wb = sW + (uint32_t)(s % WS) * kStageBytes;
    b_hi = wg_desc_sw128(wb);
    b_lo = wg_desc_sw128(wb + NC * 128u);
  };

  if constexpr (MODE == 4) {
    // ---- LinearSE3 (reference S:78-95): rows = (node, m) of x [nodes, D, M], A[row, d] = x[node, d, m] read in place (stride
    // M), chunk c of stage s = input channels 64 s + 16 c .. +15; out[node, o, m] (+ residual) in the reference layout
    const ZSeg& z = prm.seg[0];
    const int M = z.ncomp, Dn = z.Ci;
    int64_t node[2];
    int m[2];
    float sc[2];
    const float* xrow[2];
#pragma unroll
    for (int rs = 0; rs < 2; ++rs) {
      node[rs] = live[rs] ? eg[rs] / M : 0;
      m[rs] = live[rs] ? (int)(eg[rs] - node[rs] * M) : 0;
      sc[rs] = live[rs] ? prm.sx[node[rs]] : 1.f;
      xrow[rs] = z.X + ((size_t)node[rs] * Dn) * M + m[rs];
    }
    for (int s = 0; s < S; ++s) {
      float v[4][2][4];
#pragma unroll
      for (int c = 0; c < 4; ++c)
#pragma unroll
        for (int rs = 0; rs < 2; ++rs)
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int d = 64 * s + 16 * c + kq + (q & 1) + 8 * (q >> 1);
            v[c][rs][q] = live[rs] ? __ldg(xrow[rs] + (size_t)d * M) * sc[rs] : 0.f;
          }
      uint64_t b_hi, b_lo;
      wait_stage(s, b_hi, b_lo);
      uint32_t hi[4][4], lo[4][4];
#pragma unroll
      for (int c = 0; c < 4; ++c) z_frag(v[c], hi[c], lo[c]);
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < 4; ++c) z_mma3<NR>(D[0], hi[c], lo[c], b_hi + 2 * c, b_lo + 2 * c);
      finish_stage(s);
    }
#pragma unroll
    for (int rs = 0; rs < 2; ++rs) {
      if (!live[rs]) continue;
      const float inv = 1.f / sc[rs];
      const int64_t Eo = prm.out_es;                            // output channels of the layer
      const size_t o0 = (size_t)nt * N + (size_t)hs * NC + kq;
      float* dst = prm.out + ((size_t)node[rs] * Eo + o0) * M + m[rs];
      const float* res = z.U ? z.U + ((size_t)node[rs] * Eo + o0) * M + m[rs] : nullptr;
#pragma unroll
      for (int g = 0; g < NC / 8; ++g)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          const size_t o = (size_t)(8 * g + b) * M;
          dst[o] = acc[0][4 * g + 2 * rs + b] * inv + (res ? __ldg(res + o) : 0.f);
        }
    }
  } else {
    // ---- MODE 1 / 2 / 3.  (C_in F) % 4 == 0: every chunk of a stage is valid; X is padded to whole edge tiles, so rows past E
    // are readable
    int s = 0;                                 // global stage index
    for (int sg = 0; sg < prm.n_seg; ++sg) {
      const ZSeg& z = prm.seg[sg];
      const int ns = z.n_stage;
      const size_t istride = (size_t)z.ncomp * 128;                     // floats between consecutive input channels of X
      const float* xp = z.X + ((size_t)mt * z.Ci * z.ncomp + z.cplus) * 128 + r0;
      const float* xm = z.X + ((size_t)mt * z.Ci * z.ncomp + z.cminus) * 128 + r0;
#pragma unroll
      for (int rs = 0; rs < 2; ++rs) {
        const float* urow = z.U + (size_t)(live[rs] ? eg[rs] : 0) * 64;
#pragma unroll
        for (int q = 0; q < 4; ++q) u[rs][q] = live[rs] ? __ldg(urow + kq + (q & 1) + 8 * (q >> 1)) * sxe[rs] : 0.f;
      }
      if constexpr (MODE == 1) {
        // chunk c of stage sl = input channel 4 sl + c; its rows are loaded one stage ahead, as soon as the chunk is generated
        float y[4][2];
#pragma unroll
        for (int c = 0; c < 4; ++c)
#pragma unroll
          for (int rs = 0; rs < 2; ++rs) y[c][rs] = __ldg(xp + c * istride + 8 * rs);
#pragma unroll 1
        for (int sl = 0; sl < ns; ++sl, ++s) {
          const float* xn = (sl + 1 < ns) ? xp + 4 * istride : xp;    // the last stage reloads its own rows, never past the tile
          uint64_t b_hi, b_lo;
          wait_stage(s, b_hi, b_lo);
          static_for<4>([&](auto cc) {
            constexpr int C = decltype(cc)::value;
            chunk_mma(cc, ic<0>(), s, y[C], b_hi, b_lo);
#pragma unroll
            for (int rs = 0; rs < 2; ++rs) y[C][rs] = __ldg(xn + C * istride + 8 * rs);
          });
          end_stage(s);
          xp = xn;
        }
      } else if constexpr (MODE == 2) {
#pragma unroll 1
        for (int sl = 0; sl < ns; ++sl, ++s) {
          // input channels 2 sl + il; chunk 2 il + f, f in (a, b).  component +m: (a: U x+), (b: -U x-); component -m: (a: U x-), (b: U x+)
          float yp[2][2], ym[2][2];
#pragma unroll
          for (int il = 0; il < 2; ++il)
#pragma unroll
            for (int rs = 0; rs < 2; ++rs) {
              const size_t o = (size_t)(2 * sl + il) * istride + 8 * rs;
              yp[il][rs] = __ldg(xp + o);
              ym[il][rs] = __ldg(xm + o);
            }
          uint64_t b_hi, b_lo;
          wait_stage(s, b_hi, b_lo);
          uint32_t hp[2][4], lp[2][4], hm[2][4], lm[2][4];
#pragma unroll
          for (int il = 0; il < 2; ++il) {
            zf(yp[il], hp[il], lp[il]);
            zf(ym[il], hm[il], lm[il]);
          }
          uint32_t hn[2][4], ln[2][4];         // -U x-
#pragma unroll
          for (int il = 0; il < 2; ++il)
#pragma unroll
            for (int q = 0; q < 4; ++q) { hn[il][q] = hm[il][q] ^ 0x80008000u; ln[il][q] = lm[il][q] ^ 0x80008000u; }
          wgmma_fence();
#pragma unroll
          for (int il = 0; il < 2; ++il) {
            const uint64_t ba_hi = b_hi + 2 * (2 * il), ba_lo = b_lo + 2 * (2 * il);
            const uint64_t bb_hi = b_hi + 2 * (2 * il + 1), bb_lo = b_lo + 2 * (2 * il + 1);
            z_mma3<NR>(D[0], hp[il], lp[il], ba_hi, ba_lo);
            z_mma3<NR>(D[0], hn[il], ln[il], bb_hi, bb_lo);
            z_mma3<NR>(D[NA - 1], hm[il], lm[il], ba_hi, ba_lo);
            z_mma3<NR>(D[NA - 1], hp[il], lp[il], bb_hi, bb_lo);
          }
          finish_stage(s);
        }
      } else {
        // K chunk q = 4 sl + c of the segment: input channel q / 3, weight set q % 3 of (a+b, a, b) <-> y = (c, d - c, c + d).  The
        // map repeats every 3 stages (12 chunks, 4 input channels) and ns = 3 C_in / 4, so the loop runs over whole periods with
        // every channel offset and accumulator index known at compile time.  Each (channel, +-m component, row) value is loaded
        // once per period, one period ahead: channel j of the next period as soon as the last chunk of channel j is generated.
        const int dmo = (z.cminus - z.cplus) * 128;                   // from x'(+m) to x'(-m) of the same channel
        float x[4][2][2];                      // [channel of the period][c = x'(+m), d = x'(-m)][row]
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int rs = 0; rs < 2; ++rs) {
            x[j][0][rs] = __ldg(xp + j * istride + 8 * rs);
            x[j][1][rs] = __ldg(xp + dmo + j * istride + 8 * rs);
          }
        const int np = ns / 3;
#pragma unroll 1
        for (int p = 0; p < np; ++p) {
          const size_t adv = (p + 1 < np) ? 4 * istride : 0;          // the last period reloads its own rows, never past the tile
          static_for<3>([&](auto tc) {
            uint64_t b_hi, b_lo;
            wait_stage(s, b_hi, b_lo);
            static_for<4>([&](auto cc) {
              constexpr int Q = 4 * decltype(tc)::value + decltype(cc)::value, J = Q / 3, T = Q % 3;
              float y[2];
#pragma unroll
              for (int rs = 0; rs < 2; ++rs) {
                const float cp = x[J][0][rs], dm = x[J][1][rs];
                y[rs] = (T == 0) ? cp : (T == 1) ? (dm - cp) : (cp + dm);
              }
              chunk_mma(cc, ic<T>(), s, y, b_hi, b_lo);
              if constexpr (T == 2) {
#pragma unroll
                for (int rs = 0; rs < 2; ++rs) {
                  x[J][0][rs] = __ldg(xp + adv + J * istride + 8 * rs);
                  x[J][1][rs] = __ldg(xp + adv + dmo + J * istride + 8 * rs);
                }
              }
            });
            end_stage(s);
            ++s;
          });
          xp += adv;
        }
      }
    }

    // out'[e, component plane, channels of this CTA]
#pragma unroll
    for (int rs = 0; rs < 2; ++rs) {
      if (!live[rs]) continue;
      const float inv = 1.f / sxe[rs];
#pragma unroll
      for (int a = 0; a < NO; ++a) {
        float* dst = prm.out + (size_t)eg[rs] * prm.out_es + prm.comp_off[a] + (size_t)nt * N + (size_t)hs * NC + kq;
#pragma unroll
        for (int g = 0; g < NC / 8; ++g)
          *reinterpret_cast<float2*>(dst + 8 * g) = make_float2(acc[a][4 * g + 2 * rs] * inv, acc[a][4 * g + 2 * rs + 1] * inv);
      }
    }
  }
}

// Weight image of one sub-segment: rows (o, i, f) of Fp (columns [col0, col0+16) of each row) -> stages [stage0, stage0+n) of
// the launch image.  Chunk c = i*F + f of the segment sits in stage c/4 at K columns [(c%4)*16, +16).
// gauss != 0 (MODE 3): Fp rows are (o, i, f in {a, b}); K chunk q = 4 sl + c of the segment = weight set q % 3 of (a+b, a, b) of
// input channel q / 3.
__global__ void zpack_kernel(const float* __restrict__ Fp, int Kp, int col0, int Co, int CiF, int N, int S, int stage0, int n_stage,
                             int gauss, uint8_t* __restrict__ img) {
  const int nt = blockIdx.y, sl = blockIdx.x;
  uint8_t* dst = img + ((size_t)nt * S + stage0 + sl) * (2u * N * 128u);
  for (int t = threadIdx.x; t < N * 64; t += blockDim.x) {
    const int r = t >> 6, k = t & 63;
    const int o = nt * N + r;
    float w = 0.f;
    if (gauss) {
      const int q = sl * 4 + (k >> 4);
      const int ty = q % 3, i = q / 3;
      if (2 * i + 1 < CiF && o < Co) {
        const float wa = Fp[((size_t)o * CiF + 2 * i) * Kp + col0 + (k & 15)], wb = Fp[((size_t)o * CiF + 2 * i + 1) * Kp + col0 + (k & 15)];
        w = (ty == 0) ? wa + wb : (ty == 1) ? wa : wb;
      }
    } else {
      const int c = sl * 4 + (k >> 4);
      if (c < CiF && o < Co) w = Fp[((size_t)o * CiF + c) * Kp + col0 + (k & 15)];
    }
    const __half hi = __float2half_rn(w);
    const __half lo = __float2half_rn(w - __half2float(hi));
    const uint32_t off = (uint32_t)(r * 128 + (((k >> 3) ^ (r & 7)) << 4) + (k & 7) * 2);
    *reinterpret_cast<__half*>(dst + off) = hi;
    *reinterpret_cast<__half*>(dst + (size_t)N * 128 + off) = lo;
  }
}

template <int MODE, int N, int NC>
static int launch_z(const ZParams& prm, cudaStream_t s) {
  constexpr uint32_t kStageBytes = 2u * NC * 128u;
  constexpr int WS = (kZWRingBytes / kStageBytes > 8) ? 8 : (int)(kZWRingBytes / kStageBytes);
  const size_t smem = 1024 + (size_t)WS * kStageBytes + 256;
  auto kern = zgemm_kernel<MODE, N, NC>;
  SE3_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t grid = (int64_t)prm.n_mt * prm.n_nt * (N / NC);
  SE3_REQUIRE(grid < 2147483647ll, "se3_zgemm: grid too large");
  kern<<<(unsigned)grid, kZThreads, smem, s>>>(prm);
  SE3_LAUNCH_OK();
  return SE3_OK;
}

static int z_env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v ? atoi(v) : dflt;
}

}  // namespace se3

extern "C" int se3_zgemm_tile_n(int Co, int mode) {
  if (Co <= 0 || Co % 128 != 0) return -1;
  if (mode == 2 || mode == 3 || mode == 4) return 128;
  if (mode != 1) return -1;
  return (Co % 256 == 0) ? 256 : 128;
}

extern "C" int64_t se3_zgemm_image_bytes(int Co, int mode, int total_stages) {
  const int N = se3_zgemm_tile_n(Co, mode);
  if (N < 0 || total_stages <= 0) return -1;
  return (int64_t)(Co / N) * total_stages * 2 * N * 128;
}

extern "C" int se3_zgemm_pack(const float* Fp, int Kp, int col0, int Co, int CiF, int mode, int total_stages, int stage0, void* image,
                              void* stream) {
  using namespace se3;
  const int N = se3_zgemm_tile_n(Co, mode);
  SE3_REQUIRE(N > 0, "se3_zgemm_pack: Co=%d must be a multiple of 128 (mode %d)", Co, mode);
  SE3_REQUIRE(Fp != nullptr && image != nullptr, "se3_zgemm_pack: null pointer");
  SE3_REQUIRE(Kp >= 16 && Kp % 16 == 0 && col0 >= 0 && col0 + 16 <= Kp, "se3_zgemm_pack: bad column range");
  SE3_REQUIRE(CiF > 0 && (mode == 1 || CiF % 2 == 0), "se3_zgemm_pack: bad sizes");
  // mode 3: three weight sets (a+b, a, b) of 4 input channels per stage; modes 1, 2: 4 rows (i,f) per stage
  const int n_stage = (mode == 3) ? 3 * (int)ceil_div(CiF / 2, 4) : (int)ceil_div(CiF, 4);
  SE3_REQUIRE(stage0 >= 0 && stage0 + n_stage <= total_stages, "se3_zgemm_pack: stage range outside the image");
  zpack_kernel<<<dim3((unsigned)n_stage, (unsigned)(Co / N)), 256, 0, as_stream(stream)>>>(Fp, Kp, col0, Co, CiF, N, total_stages, stage0, n_stage,
                                                                                         mode == 3 ? 1 : 0, reinterpret_cast<uint8_t*>(image));
  SE3_LAUNCH_OK();
  return SE3_OK;
}

// LinearSE3 on the tensor cores (reference S:78-95): out[node, o, m] = sum_d x[node, d, m] W[d, o] (+ res[node, o, m]) with the A
// operand read in place from the reference layout (row = (node, m), stride M), split to fp16 hi / lo on the fly; the same
// pipeline as se3_zgemm_fwd (MODE 4: one N = 128 accumulator, fp32 drain).  w_img = se3_zgemm_pack(W^T viewed [Eo * D/16, 16],
// Kp 16, col0 0, Co Eo, CiF D/16, mode 4).  sx [nodes]: power-of-two scale per node (se3_node_scale_fwd).
extern "C" int se3_linear_tc_fwd(const float* x, const void* w_img, const float* res, const float* sx, int64_t nodes, int D, int Eo,
                                 int M, float* out, void* stream) {
  using namespace se3;
  SE3_REQUIRE(nodes > 0 && M >= 1 && M <= 11, "se3_linear_tc_fwd: bad sizes");
  SE3_REQUIRE(D > 0 && D % 64 == 0 && Eo > 0 && Eo % 128 == 0, "se3_linear_tc_fwd: D=%d must be a multiple of 64 and Eo=%d of 128", D, Eo);
  SE3_REQUIRE(x != nullptr && w_img != nullptr && sx != nullptr && out != nullptr, "se3_linear_tc_fwd: null pointer");
  ZParams prm;
  prm.n_seg = 1;
  prm.seg[0].U = res;
  prm.seg[0].X = x;
  prm.seg[0].Ci = D;
  prm.seg[0].ncomp = M;
  prm.seg[0].cplus = prm.seg[0].cminus = 0;
  prm.seg[0].n_stage = D / 64;
  prm.seg[0].pad = 0;
  prm.w_img = reinterpret_cast<const uint8_t*>(w_img);
  prm.sx = sx;
  prm.out = out;
  prm.E = nodes * M;
  prm.out_es = Eo;
  prm.comp_off[0] = prm.comp_off[1] = 0;
  prm.n_mt = (int)ceil_div(prm.E, SE3_TILE_E);
  prm.n_nt = Eo / 128;
  prm.S = D / 64;
  prm.flush_stages = std::max(1, z_env_int("SE3B200_Z_FLUSH", 8));
  return launch_z<4, 128, 128>(prm, as_stream(stream));
}

extern "C" int se3_zgemm_fwd(const se3_zseg* segs, int n_seg, const void* w_img, const float* sx, int64_t E, int Co, int mode,
                             float* out, int64_t out_edge_stride, int comp_off0, int comp_off1, int flush_stages, void* stream) {
  using namespace se3;
  const int N = se3_zgemm_tile_n(Co, mode);
  SE3_REQUIRE(N > 0 && mode != 4, "se3_zgemm_fwd: Co=%d must be a multiple of 128 and mode 1, 2 or 3 (got %d)", Co, mode);
  SE3_REQUIRE(E > 0 && n_seg >= 1 && n_seg <= kZMaxSeg, "se3_zgemm_fwd: bad sizes (1..%d segments)", kZMaxSeg);
  SE3_REQUIRE(segs != nullptr && w_img != nullptr && sx != nullptr && out != nullptr, "se3_zgemm_fwd: null pointer");
  SE3_REQUIRE(out_edge_stride >= Co && out_edge_stride % 4 == 0 && comp_off0 % 4 == 0 && comp_off1 % 4 == 0 &&
              (reinterpret_cast<uintptr_t>(out) & 15) == 0, "se3_zgemm_fwd: output rows must be 16-byte aligned");
  ZParams prm;
  prm.n_seg = n_seg;
  int S = 0;
  const int F = (mode == 1) ? 1 : 2;          // MODE 1: one weight per (o,i); MODE 2 / 3: the pair (a, b)
  for (int i = 0; i < n_seg; ++i) {
    const se3_zseg& z = segs[i];
    SE3_REQUIRE(z.U != nullptr && z.X != nullptr && z.Ci > 0 && z.ncomp >= 1 && z.cplus >= 0 && z.cplus < z.ncomp &&
                z.cminus >= 0 && z.cminus < z.ncomp, "se3_zgemm_fwd: bad segment %d", i);
    SE3_REQUIRE((z.Ci * F) % 4 == 0 && (mode != 3 || z.Ci % 4 == 0), "se3_zgemm_fwd: C_in * F = %d must be a multiple of 4 (mode 3: C_in % 4 == 0)", z.Ci * F);
    prm.seg[i].U = z.U;
    prm.seg[i].X = z.X;
    prm.seg[i].Ci = z.Ci;
    prm.seg[i].ncomp = z.ncomp;
    prm.seg[i].cplus = z.cplus;
    prm.seg[i].cminus = z.cminus;
    prm.seg[i].n_stage = (mode == 3) ? 3 * (z.Ci / 4) : z.Ci * F / 4;
    prm.seg[i].pad = 0;
    S += prm.seg[i].n_stage;
  }
  prm.w_img = reinterpret_cast<const uint8_t*>(w_img);
  prm.sx = sx;
  prm.out = out;
  prm.E = E;
  prm.out_es = out_edge_stride;
  prm.comp_off[0] = comp_off0;
  prm.comp_off[1] = comp_off1;
  prm.n_mt = (int)ceil_div(E, SE3_TILE_E);
  prm.n_nt = Co / N;
  prm.S = S;
  // default drain period: 96 accumulating K = 16 MMAs per accumulator (8 stages of 12; mode 3 spreads its stages over three
  // accumulators): rel. error 4e-6 against float64 for all-positive operands at K = 65536 (2.5e-4 if never drained)
  prm.flush_stages = std::max(1, flush_stages > 0 ? flush_stages
                                                     : z_env_int("SE3B200_Z_FLUSH", mode == 3 ? 24 : 8) * std::max(1, z_env_int("SE3B200_Z_FLUSH_MULT", 1)));
  cudaStream_t s = as_stream(stream);
  if (mode == 3) return launch_z<3, 128, 64>(prm, s);
  if (mode == 2) return launch_z<2, 128, 64>(prm, s);
  return N == 256 ? launch_z<1, 256, 128>(prm, s) : launch_z<1, 128, 128>(prm, s);
}
