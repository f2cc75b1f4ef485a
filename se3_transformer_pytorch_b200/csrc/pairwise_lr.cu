// K4 (tensor cores, low-rank radial path): the fused pairwise kernel when the radial-trunk outputs of a pair,
// G = [g(e)]_e in R^{E x 128}, are numerically low rank.
//
// For distance-only radial functions (no per-edge features besides r_ij: BASELINE cfg1/2/3/5) every row of G is a point
// on a smooth one-parameter curve g(|r_ij|), and G has numerical rank ~16 to 1e-7 (DESIGN.md section 4.2).
// The host factors  G ~= U V^T  (U: E x r, V: 128 x r orthonormal, residual verified every forward) and folds V into the
// last radial layer:
//     R[e,(o,i,f)] = W3[(o,i,f),:] . g[e,:] + b3  =  [U[e,:], 1] . [F'[(o,i,f),:], b3]      with F' = W3 V  (N x r)
// so the dense contraction has K = r+1 <= 64 instead of 128 and the bias rides along as one more K column.  Everything
// downstream is unchanged:   out[e,o,p] (+)= sum_{i,f} R[e,o,i,f] * T[e,i,f,p]   (reference S:294-299, 326-343, 251-254).
//
// The kernel is the one of pairwise_wg.cuh (128 edges x 32 channels per CTA, wgmma with A = U hi / lo and B = F' hi / lo in
// shared memory, contraction with T from the accumulator registers).  It serves fibers that are not multiples of 128
// channels; the production path of wider fibers is csrc/zgemm.cu (DESIGN.md 4.5).
#include "common.cuh"
#include "pairwise_wg.cuh"
#include <cuda_fp16.h>

namespace se3 {

constexpr uint32_t kLrUnitBytes = kPwUnitBytes;   // one W unit: [hi 16 KiB | lo 16 KiB], K padded to 64

// F'' image packer: Fp fp32 [Co*Ci*F, Kp] (columns 0..r-1 = W3 V, column r = b3, rest 0) -> per 32-channel block a row of
// 32 KiB units [hi 128 x 64 | lo 128 x 64] fp16, SW128, row = if_local*32 + o_local.  A unit holds spu = 64 / Kp (Kp = 16,
// 32: 4, 2; else 1) consecutive (i,f) steps side by side along K: step j of the unit occupies K columns [j*Kp, (j+1)*Kp),
// so the streamed bytes per step are what the MMAs read (K = Kp), not a K = 64 padded tile.
__global__ void pack_lr_kernel(const float* __restrict__ Fp, int Co, int CiF, int NU, int Kp, int spu, uint8_t* __restrict__ img) {
  const int64_t tile = blockIdx.x;
  const int ob = (int)(tile / NU), un = (int)(tile % NU);
  uint8_t* dst = img + (size_t)tile * kLrUnitBytes;
  for (int t = threadIdx.x; t < 128 * 64; t += blockDim.x) {
    const int r = t >> 6, k = t & 63;
    const int sub = k / Kp, kk = k - sub * Kp;
    const int ifb = un * spu + sub;
    const int o = ob * SE3_TILE_O + (r & 31), ifx = ifb * SE3_TILE_IF + (r >> 5);
    const float w = (sub < spu && ifx < CiF) ? Fp[((size_t)o * CiF + ifx) * Kp + kk] : 0.f;
    const __half hi = __float2half_rn(w);
    const __half lo = __float2half_rn(w - __half2float(hi));
    const uint32_t off = sw128_off(r, k);
    *reinterpret_cast<__half*>(dst + off) = hi;
    *reinterpret_cast<__half*>(dst + kSubBytes + off) = lo;
  }
}

__host__ __device__ inline int lr_steps_per_unit(int Kp) { return Kp == 16 ? 4 : Kp == 32 ? 2 : 1; }

}  // namespace se3

extern "C" int64_t se3_lowrank_image_bytes(int Co, int Ci, int F, int Kp) {
  if (Co <= 0 || Ci <= 0 || F <= 0 || Co % SE3_TILE_O != 0 || Kp < 16 || Kp > 64 || Kp % 16 != 0) return -1;
  const int64_t NIFB = se3::ceil_div((int64_t)Ci * F, SE3_TILE_IF);
  const int64_t NU = se3::ceil_div(NIFB, (int64_t)se3::lr_steps_per_unit(Kp));
  return (int64_t)(Co / SE3_TILE_O) * NU * se3::kLrUnitBytes;
}

extern "C" int se3_pack_lowrank(const float* Fp, int Co, int Ci, int F, int Kp, void* image, void* stream) {
  using namespace se3;
  SE3_REQUIRE(Co > 0 && Ci > 0 && F > 0 && Co % SE3_TILE_O == 0, "se3_pack_lowrank: Co must be a positive multiple of %d", SE3_TILE_O);
  SE3_REQUIRE(Kp >= 16 && Kp <= 64 && Kp % 16 == 0, "se3_pack_lowrank: Kp=%d must be 16, 32, 48 or 64", Kp);
  const int CiF = Ci * F;
  const int NIFB = (int)ceil_div(CiF, SE3_TILE_IF);
  const int spu = lr_steps_per_unit(Kp);
  const int NU = (int)ceil_div(NIFB, spu);
  const int64_t tiles = (int64_t)(Co / SE3_TILE_O) * NU;
  SE3_REQUIRE(tiles < 2147483647ll, "se3_pack_lowrank: too many tiles");
  pack_lr_kernel<<<(unsigned)tiles, 256, 0, as_stream(stream)>>>(Fp, Co, CiF, NU, Kp, spu, reinterpret_cast<uint8_t*>(image));
  SE3_LAUNCH_OK();
  return SE3_OK;
}

extern "C" int se3_pairwise_lr_fwd(const float* U, const void* w_img, const float* T, int64_t E, int Co, int Ci, int F, int P,
                                   int Kp, int accumulate, float* out, void* stream) {
  using namespace se3;
  SE3_REQUIRE(E > 0 && Co > 0 && Ci > 0 && F > 0, "se3_pairwise_lr_fwd: bad sizes");
  SE3_REQUIRE(Co % SE3_TILE_O == 0, "se3_pairwise_lr_fwd: Co=%d must be a multiple of %d", Co, SE3_TILE_O);
  SE3_REQUIRE(P == 1 || P == 2 || P == 3 || P == 5 || P == 7, "se3_pairwise_lr_fwd: P=%d unsupported (1, 2, 3, 5, 7)", P);
  SE3_REQUIRE(Kp >= 16 && Kp <= 64 && Kp % 16 == 0, "se3_pairwise_lr_fwd: Kp=%d must be 16, 32, 48 or 64", Kp);
  SE3_REQUIRE(ceil_div(E, SE3_TILE_E) * (Co / SE3_TILE_O) < 2147483647ll, "se3_pairwise_lr_fwd: grid too large");
  PwParams prm = {};
  prm.A = U;
  prm.lda = 64;
  prm.w_img = reinterpret_cast<const uint8_t*>(w_img);
  prm.T = T;
  prm.out = out;
  prm.E = E;
  prm.NIFB = (int)ceil_div((int64_t)Ci * F, SE3_TILE_IF);
  prm.n_mt = (int)ceil_div(E, SE3_TILE_E);
  prm.n_ob = Co / SE3_TILE_O;
  prm.accumulate = accumulate;
  prm.nk16 = Kp / 16;
  prm.out_es = (int64_t)Co * P;
  prm.out_os = P;
  for (int p = 0; p < 7; ++p) prm.p_off[p] = p;
  prm.spu = lr_steps_per_unit(Kp);
  prm.NU = (int)ceil_div((int64_t)prm.NIFB, (int64_t)prm.spu);
  cudaStream_t s = as_stream(stream);
  switch (P) {
    case 1: return launch_pw<1, false, false, 4>(prm, s);
    case 2: return launch_pw<2, false, false, 4>(prm, s);
    case 3: return launch_pw<3, false, false, 4>(prm, s);
    case 5: return launch_pw<5, false, false, 4>(prm, s);
    default: return launch_pw<7, false, false, 4>(prm, s);
  }
}
