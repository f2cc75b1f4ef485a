// K4a: T[e,i,f,p] = sum_q basis[e,p,q,f] * x[b(e), idx[e], i, q]
//
// This is the neighbour gather of ConvSE3 (se3_transformer_pytorch.py:237-238, utils.py:56-70) fused with the
// basis half of PairwiseConv's kernel (S:336-338) in the factored form of SURVEY.md A.4: the per-edge
// [Co(2lo+1) x Ci(2li+1)] kernel is never formed.  T is shared by every ConvSE3 that reads the same input
// features (to_k and to_v of one attention block), and is written once in the tile layout the pairwise kernels
// stream:  [edge tile (128)][if-block][if_local (4)][p-quad][edge_local (128)][4 floats],  if = i*F + f.
#include "common.cuh"

namespace se3 {

constexpr int kTE = SE3_TILE_E;

// One CTA = one edge tile x a slab of `ci_per_cta` input channels; thread = edge.
__global__ void __launch_bounds__(kTE)
tbuild_kernel(const float* __restrict__ x, const int64_t* __restrict__ idx, const float* __restrict__ basis,
              int64_t E, int64_t mt_begin, int n, int k, int Ci, int P, int Q, int F, int ci_per_cta,
              float* __restrict__ T) {
  extern __shared__ float Bs[];            // [P*Q][kTE]  slice of the basis for the current f
  const int el = threadIdx.x;
  const int64_t mt = blockIdx.x;                      // tile index inside the requested edge range
  const int64_t e = (mt_begin + mt) * kTE + el;       // global edge
  const bool valid = e < E;
  const int PH = (P + 3) >> 2;
  const int CiF = Ci * F;
  const int NIFB = (CiF + SE3_TILE_IF - 1) / SE3_TILE_IF;
  const int i0 = blockIdx.y * ci_per_cta;
  const int i1 = min(Ci, i0 + ci_per_cta);

  const float* xrow = nullptr;
  if (valid) {
    const int64_t bn = e / k;              // b*n + i
    const int64_t bb = bn / n;
    xrow = x + ((size_t)(bb * n + idx[e]) * Ci) * Q;
  }
  float4* Tt = reinterpret_cast<float4*>(T) + (size_t)mt * NIFB * SE3_TILE_IF * PH * kTE;

  for (int f = 0; f < F; ++f) {
    __syncthreads();
    if (valid) {
      const float* bp = basis + (size_t)e * P * Q * F + f;
      for (int pq = 0; pq < P * Q; ++pq) Bs[pq * kTE + el] = bp[(size_t)pq * F];
    }
    __syncthreads();
    for (int i = i0; i < i1; ++i) {
      float xv[11];
#pragma unroll
      for (int q = 0; q < 11; ++q) xv[q] = (valid && q < Q) ? xrow[(size_t)i * Q + q] : 0.f;
      const int ifx = i * F + f;
      float4* dst = Tt + ((size_t)(ifx / SE3_TILE_IF) * SE3_TILE_IF + (ifx % SE3_TILE_IF)) * PH * kTE + el;
      for (int ph = 0; ph < PH; ++ph) {
        float o[4] = {0.f, 0.f, 0.f, 0.f};
        if (valid) {
#pragma unroll
          for (int pp = 0; pp < 4; ++pp) {
            const int p = ph * 4 + pp;
            if (p < P) {
              float acc = 0.f;
#pragma unroll
              for (int q = 0; q < 11; ++q)
                if (q < Q) acc = fmaf(Bs[(p * Q + q) * kTE + el], xv[q], acc);
              o[pp] = acc;
            }
          }
        }
        dst[(size_t)ph * kTE] = make_float4(o[0], o[1], o[2], o[3]);
      }
    }
  }
  // zero the padded (if) slots of the last if-block (once, by the CTA that owns the last channel slab)
  if (blockIdx.y == gridDim.y - 1) {
    for (int ifx = CiF; ifx < NIFB * SE3_TILE_IF; ++ifx) {
      float4* dst = Tt + ((size_t)(ifx / SE3_TILE_IF) * SE3_TILE_IF + (ifx % SE3_TILE_IF)) * PH * kTE + el;
      for (int ph = 0; ph < PH; ++ph) dst[(size_t)ph * kTE] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}

// Fast variant for degrees <= 3.  The whole per-edge basis block ([P][Q][F] floats x 128 edges, <= 172 KiB) is staged
// in shared memory once per CTA as Bs[r][edge]; thread = (edge, channel lane).  Each input channel row x[j, i, :] is
// gathered exactly once (Q registers) and produces all F * ceil(P/4) output quads with conflict-free LDS + FMA and one
// coalesced 16-byte store per quad.
constexpr int kTbLanes = 4;     // channel lanes per edge (512 threads per CTA)

template <int P, int Q, int F>
__global__ void __launch_bounds__(kTE * kTbLanes, 1)
tbuild_reg_kernel(const float* __restrict__ x, const int64_t* __restrict__ idx, const float* __restrict__ basis,
                  int64_t E, int64_t mt_begin, int n, int k, int Ci, int ci_per_cta, float* __restrict__ T) {
  constexpr int PH = (P + 3) / 4;
  constexpr int R = P * Q * F;                           // F = 2*min(li,lo)+1 for the reference basis; 1 or 2 for caller blocks
  extern __shared__ float Bs[];                          // [R][kTE]
  const int el = threadIdx.x;
  const int lane_c = threadIdx.y;
  const int64_t mt = blockIdx.x;
  const int64_t e = (mt_begin + mt) * kTE + el;
  const bool valid = e < E;
  const int CiF = Ci * F;
  const int NIFB = (CiF + SE3_TILE_IF - 1) / SE3_TILE_IF;
  const int i0 = blockIdx.y * ci_per_cta;
  const int i1 = min(Ci, i0 + ci_per_cta);
  // stage the basis: every thread copies a quarter of its own edge's block
  {
    const float* bp = basis + (size_t)(valid ? e : 0) * R;
    for (int r = lane_c; r < R; r += kTbLanes) Bs[r * kTE + el] = valid ? bp[r] : 0.f;
  }
  const float* xrow = x;
  if (valid) {
    const int64_t bn = e / k;
    const int64_t bb = bn / n;
    xrow = x + ((size_t)(bb * n + idx[e]) * Ci) * Q;
  }
  float4* Tt = reinterpret_cast<float4*>(T) + (size_t)mt * NIFB * SE3_TILE_IF * PH * kTE + el;
  __syncthreads();
  for (int i = i0 + lane_c; i < i1; i += kTbLanes) {
    float xv[Q];
#pragma unroll
    for (int q = 0; q < Q; ++q) xv[q] = valid ? xrow[(size_t)i * Q + q] : 0.f;
#pragma unroll
    for (int f = 0; f < F; ++f) {
      const int ifx = i * F + f;
      float4* dst = Tt + ((size_t)(ifx / SE3_TILE_IF) * SE3_TILE_IF + (ifx % SE3_TILE_IF)) * PH * kTE;
#pragma unroll
      for (int ph = 0; ph < PH; ++ph) {
        float o[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int pp = 0; pp < 4; ++pp) {
          const int p = ph * 4 + pp;
          if (p < P) {
#pragma unroll
            for (int q = 0; q < Q; ++q) o[pp] = fmaf(Bs[((p * Q + q) * F + f) * kTE + el], xv[q], o[pp]);
          }
        }
        dst[(size_t)ph * kTE] = make_float4(o[0], o[1], o[2], o[3]);
      }
    }
  }
  if (blockIdx.y == gridDim.y - 1 && lane_c == 0) {
    for (int ifx = CiF; ifx < NIFB * SE3_TILE_IF; ++ifx)
      for (int ph = 0; ph < PH; ++ph)
        Tt[(((size_t)(ifx / SE3_TILE_IF) * SE3_TILE_IF + (ifx % SE3_TILE_IF)) * PH + ph) * kTE] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

template <int P, int Q, int F>
static void launch_reg(dim3 grid, cudaStream_t s, const float* x, const int64_t* idx, const float* basis, int64_t E, int64_t tb, int n,
                       int k, int Ci, int cpc, float* T) {
  const size_t smem = (size_t)P * Q * F * kTE * sizeof(float);
  cudaFuncSetAttribute(tbuild_reg_kernel<P, Q, F>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  tbuild_reg_kernel<P, Q, F><<<grid, dim3(kTE, kTbLanes), smem, s>>>(x, idx, basis, E, tb, n, k, Ci, cpc, T);
}

}  // namespace se3

extern "C" int se3_tbuild_fwd(const float* x, const int64_t* idx, const float* basis_pair, int b, int n, int k, int Ci,
                              int P, int Q, int F, int64_t tile_begin, int64_t tile_count, float* T, void* stream) {
  using namespace se3;
  SE3_REQUIRE(b > 0 && n > 0 && k > 0 && Ci > 0, "se3_tbuild_fwd: bad sizes");
  SE3_REQUIRE(P >= 1 && P <= 11 && Q >= 1 && Q <= 11 && F >= 1 && F <= 11, "se3_tbuild_fwd: degree out of range");
  const int64_t E = (int64_t)b * n * k;
  const int64_t n_all = ceil_div(E, kTE);
  SE3_REQUIRE(tile_begin >= 0 && tile_count > 0 && tile_begin + tile_count <= n_all, "se3_tbuild_fwd: tile range out of bounds");
  const int64_t n_mtiles = tile_count;
  // enough CTAs to fill the machine (132 SMs x a few CTAs) without shredding the channel loop
  int slabs = (int)std::min<int64_t>(std::max(1, Ci / 16), std::max<int64_t>(1, (132 * 2 + n_mtiles - 1) / n_mtiles));
  const int ci_per_cta = (int)ceil_div(Ci, slabs);
  slabs = (int)ceil_div(Ci, ci_per_cta);
  dim3 grid((unsigned)n_mtiles, (unsigned)slabs);
  cudaStream_t st = as_stream(stream);
  bool done = true;
#define SE3_TB(PP, QQ, FF) if (P == PP && Q == QQ && F == FF) launch_reg<PP, QQ, FF>(grid, st, x, idx, basis_pair, E, tile_begin, n, k, Ci, ci_per_cta, T); else
  // reference basis blocks: F = 2*min(li,lo)+1
  SE3_TB(1, 1, 1) SE3_TB(1, 3, 1) SE3_TB(1, 5, 1) SE3_TB(1, 7, 1) SE3_TB(3, 1, 1) SE3_TB(3, 3, 3) SE3_TB(3, 5, 3) SE3_TB(3, 7, 3)
  SE3_TB(5, 1, 1) SE3_TB(5, 3, 3) SE3_TB(5, 5, 5) SE3_TB(5, 7, 5) SE3_TB(7, 1, 1) SE3_TB(7, 3, 3) SE3_TB(7, 5, 5) SE3_TB(7, 7, 7)
  // caller blocks: gathered features (input-side contraction) and the edge-aligned (+m, -m) x (a, b) blocks
  SE3_TB(3, 3, 1) SE3_TB(2, 3, 2) SE3_TB(2, 5, 2) SE3_TB(2, 7, 2)
  { done = false; }
#undef SE3_TB
  if (done) {
  } else {
    const size_t smem = (size_t)P * Q * kTE * sizeof(float);
    SE3_CUDA_OK(cudaFuncSetAttribute(tbuild_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    tbuild_kernel<<<grid, kTE, smem, st>>>(x, idx, basis_pair, E, tile_begin, n, k, Ci, P, Q, F, ci_per_cta, T);
  }
  SE3_LAUNCH_OK();
  return SE3_OK;
}
