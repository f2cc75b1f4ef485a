// K4 (tensor cores): the fused pairwise kernel for one (degree_in, degree_out) pair of one ConvSE3.
//
//   out[e,o,p] (+)= sum_{i,f} ( W3[(o*Ci+i)*F+f,:] . g[e,:] + b3 ) * T[e,i,f,p]
//
// = RadialFunc.net.6 (se3_transformer_pytorch.py:294,299) + PairwiseConv.forward (S:326-343) + the per-edge
// mat-vec and sum over degree_in of ConvSE3.forward (S:251-254), in the factored form of SURVEY.md A.4.
//
// The only dense contraction, R = g . W3^T (M = 128 edges, N = 128 (o,i,f) columns, K = 128), runs on the Hopper tensor
// cores (wgmma m64n64k16, fp16 x fp16 -> fp32) in the kernel of pairwise_wg.cuh.  fp32 parity is kept with a 3-pass fp16
// split: g = g_hi + g_lo, W = W_hi + W_lo with hi = fp16(x), lo = fp16(x - hi): 22 mantissa bits per operand.
// R ~= g_hi W_hi + g_lo W_hi + g_hi W_lo.  fp16 range: the host only selects this kernel when |W3| and the LayerNorm-bounded
// |g| stay below 6e4 (else the fp32 SIMT kernel runs).  R never leaves the SM: the MMA warpgroups add the bias and contract
// it with the per-edge T block straight from the accumulator registers.
//
// All operands are pre-imaged in global memory in exactly the layout the kernel wants in shared memory (128-byte-swizzled
// K-major tiles; T in [if][p-quad][edge][4]) so every stage is filled by 1-D TMA bulk copies (cp.async.bulk, completion on
// mbarriers) with no tensor maps.
#include "common.cuh"
#include "pairwise_wg.cuh"
#include <cuda_fp16.h>

namespace se3 {

constexpr uint32_t kImgBytes = 2 * kPwUnitBytes;  // one 128x128 hi+lo operand image (4 sub-tiles of 16 KiB)
constexpr uint32_t kWTileBytes = kImgBytes + kPwBiasBytes;
constexpr uint32_t kUnitBytes = kPwUnitBytes;     // one k-half of a W tile: [hi 16 KiB | lo 16 KiB]

// ---------------------------------------------------------------------------------------------------------
// weight image packer: W3 fp32 [Co*Ci*F, 128] -> per (o-block, if-block) tile: [hi k0|lo k0|hi k1|lo k1|bias fp32 x128]
// ---------------------------------------------------------------------------------------------------------
__global__ void pack_w3_kernel(const float* __restrict__ W3, const float* __restrict__ b3, int Co, int CiF, int NIFB,
                               uint8_t* __restrict__ img) {
  const int64_t tile = blockIdx.x;                 // ob * NIFB + ifb
  const int ob = (int)(tile / NIFB), ifb = (int)(tile % NIFB);
  uint8_t* dst = img + (size_t)tile * kWTileBytes;
  for (int t = threadIdx.x; t < 128 * 128; t += blockDim.x) {
    const int r = t >> 7, k = t & 127;
    const int o = ob * SE3_TILE_O + (r & 31), ifx = ifb * SE3_TILE_IF + (r >> 5);
    const float w = (ifx < CiF) ? W3[((size_t)o * CiF + ifx) * SE3_RADIAL_MID + k] : 0.f;
    const __half hi = __float2half_rn(w);
    const __half lo = __float2half_rn(w - __half2float(hi));
    // W tile image: [k-half 0: hi | lo][k-half 1: hi | lo], each sub-tile 128 rows x 64 fp16, SW128
    const uint32_t off = (uint32_t)(k >> 6) * kUnitBytes + sw128_off(r, k & 63);
    *reinterpret_cast<__half*>(dst + off) = hi;
    *reinterpret_cast<__half*>(dst + kSubBytes + off) = lo;
    if (k == 0) reinterpret_cast<float*>(dst + kImgBytes)[r] = (ifx < CiF) ? b3[(size_t)o * CiF + ifx] : 0.f;
  }
}

template <bool kDumpR>
static int dispatch_tc(const float* g, const void* w_img, const float* T, int64_t E, int Co, int Ci, int F, int P,
                       int accumulate, float* out, float* dumpR, void* stream) {
  SE3_REQUIRE(E > 0 && Co > 0 && Ci > 0 && F > 0, "se3_pairwise_tc_fwd: bad sizes");
  SE3_REQUIRE(Co % SE3_TILE_O == 0, "se3_pairwise_tc_fwd: Co=%d must be a multiple of %d (use the SIMT kernel)", Co, SE3_TILE_O);
  SE3_REQUIRE(P == 1 || P == 3 || P == 5 || P == 7, "se3_pairwise_tc_fwd: P=%d unsupported (degree_out <= 3)", P);
  SE3_REQUIRE(ceil_div(E, SE3_TILE_E) * (Co / SE3_TILE_O) < 2147483647ll, "se3_pairwise_tc_fwd: grid too large");
  PwParams prm = {};
  prm.A = g;
  prm.lda = SE3_RADIAL_MID;
  prm.w_img = reinterpret_cast<const uint8_t*>(w_img);
  prm.T = T;
  prm.out = out;
  prm.dumpR = dumpR;
  prm.E = E;
  prm.NIFB = (int)ceil_div((int64_t)Ci * F, SE3_TILE_IF);
  prm.n_mt = (int)ceil_div(E, SE3_TILE_E);
  prm.n_ob = Co / SE3_TILE_O;
  prm.accumulate = accumulate;
  prm.nk16 = 8;
  prm.spu = 1;
  prm.NU = 2 * prm.NIFB;
  prm.out_es = (int64_t)Co * P;
  prm.out_os = P;
  for (int p = 0; p < 7; ++p) prm.p_off[p] = p;
  cudaStream_t s = as_stream(stream);
  switch (P) {
    case 1: return launch_pw<1, true, kDumpR, 3>(prm, s);
    case 3: return launch_pw<3, true, kDumpR, 3>(prm, s);
    case 5: return launch_pw<5, true, kDumpR, 3>(prm, s);
    default: return launch_pw<7, true, kDumpR, 3>(prm, s);
  }
}

}  // namespace se3

extern "C" int64_t se3_w3_image_bytes(int Co, int Ci, int F) {
  if (Co <= 0 || Ci <= 0 || F <= 0 || Co % SE3_TILE_O != 0) return -1;
  const int64_t NIFB = se3::ceil_div((int64_t)Ci * F, SE3_TILE_IF);
  return (int64_t)(Co / SE3_TILE_O) * NIFB * se3::kWTileBytes;
}

extern "C" int se3_pack_w3(const float* W3, const float* b3, int Co, int Ci, int F, void* image, void* stream) {
  using namespace se3;
  SE3_REQUIRE(Co > 0 && Ci > 0 && F > 0 && Co % SE3_TILE_O == 0, "se3_pack_w3: Co must be a positive multiple of %d", SE3_TILE_O);
  const int CiF = Ci * F;
  const int NIFB = (int)ceil_div(CiF, SE3_TILE_IF);
  const int64_t tiles = (int64_t)(Co / SE3_TILE_O) * NIFB;
  SE3_REQUIRE(tiles < 2147483647ll, "se3_pack_w3: too many tiles");
  pack_w3_kernel<<<(unsigned)tiles, 256, 0, as_stream(stream)>>>(W3, b3, Co, CiF, NIFB, reinterpret_cast<uint8_t*>(image));
  SE3_LAUNCH_OK();
  return SE3_OK;
}

extern "C" int se3_pairwise_tc_fwd(const float* g, const void* w_img, const float* T, int64_t E, int Co, int Ci, int F,
                                   int P, int accumulate, float* out, void* stream) {
  return se3::dispatch_tc<false>(g, w_img, T, E, Co, Ci, F, P, accumulate, out, nullptr, stream);
}

// Diagnostic (tests only): same kernel, additionally dumps R + bias of step 0 as [edge tiles, Co/32, 128 edges, 128 cols].
extern "C" int se3_pairwise_tc_debug(const float* g, const void* w_img, const float* T, int64_t E, int Co, int Ci, int F,
                                     int P, int accumulate, float* out, float* dumpR, void* stream) {
  return se3::dispatch_tc<true>(g, w_img, T, E, Co, Ci, F, P, accumulate, out, dumpR, stream);
}
