// K3: radial trunk -- the first six stages of RadialFunc.net (se3_transformer_pytorch.py:287-293) for all
// (degree_in, degree_out) pairs of one ConvSE3 in a single launch.  The last Linear (net.6) is NOT applied here:
// its output is consumed on-chip by the pairwise kernels.
//
// Output: g fp32 [pairs, E, 128]; the tensor-core kernel splits its 128-edge tile of g into fp16 hi/lo on the fly
// while loading it into shared memory.
#include "common.cuh"

namespace se3 {

constexpr int kMid = SE3_RADIAL_MID;  // 128
constexpr int kTrunkEB = 32;          // edges per CTA

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752440f)); }

// LayerNorm (eps 1e-5, biased variance) + GELU over the 128 hidden units of each edge; one warp per edge.
__device__ __forceinline__ void ln_gelu_rows(float (*h)[kMid + 4], int ne, const float* __restrict__ w,
                                             const float* __restrict__ bsh) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int e = warp; e < ne; e += 4) {
    float v[4];
    float s = 0.f;
#pragma unroll
    for (int t = 0; t < 4; ++t) { v[t] = h[e][lane + 32 * t]; s += v[t]; }
    const float mu = warp_sum(s) * (1.f / kMid);
    float q = 0.f;
#pragma unroll
    for (int t = 0; t < 4; ++t) { const float d = v[t] - mu; q += d * d; }
    const float rstd = rsqrtf(warp_sum(q) * (1.f / kMid) + 1e-5f);
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int c = lane + 32 * t;
      h[e][c] = gelu_erf((v[t] - mu) * rstd * w[c] + bsh[c]);
    }
  }
}

__global__ void __launch_bounds__(128)
radial_trunk_kernel(const float* __restrict__ feat, int64_t E, int in_dim, const float* __restrict__ params,
                    int64_t param_stride, float* __restrict__ out_g) {
  __shared__ __align__(16) float h[kTrunkEB][kMid + 4];
  __shared__ float fs[kTrunkEB][64];
  const int pair = blockIdx.y;
  const int64_t e0 = (int64_t)blockIdx.x * kTrunkEB;
  const int ne = (int)max((int64_t)0, min((int64_t)kTrunkEB, E - e0));
  const int t = threadIdx.x;
  const float* P = params + (size_t)pair * param_stride;
  const float* W1T = P;                       // [in_dim][128]
  const float* b1 = W1T + (size_t)in_dim * kMid;
  const float* ln1w = b1 + kMid;
  const float* ln1b = ln1w + kMid;
  const float* W2T = ln1b + kMid;             // [128][128]  (c, t)
  const float* b2 = W2T + kMid * kMid;
  const float* ln2w = b2 + kMid;
  const float* ln2b = ln2w + kMid;

  for (int idx = t; idx < ne * in_dim; idx += 128) fs[idx / in_dim][idx % in_dim] = feat[(e0 + idx / in_dim) * in_dim + idx % in_dim];
  __syncthreads();
  // layer 1: thread t = hidden unit t
  {
    float acc[kTrunkEB];
    const float bias = b1[t];
#pragma unroll
    for (int e = 0; e < kTrunkEB; ++e) acc[e] = bias;
    for (int d = 0; d < in_dim; ++d) {
      const float w = W1T[d * kMid + t];
#pragma unroll
      for (int e = 0; e < kTrunkEB; ++e) acc[e] = fmaf(fs[e][d], w, acc[e]);
    }
#pragma unroll
    for (int e = 0; e < kTrunkEB; ++e) h[e][t] = acc[e];
  }
  __syncthreads();
  ln_gelu_rows(h, ne, ln1w, ln1b);
  __syncthreads();
  // layer 2
  {
    float acc[kTrunkEB];
    const float bias = b2[t];
#pragma unroll
    for (int e = 0; e < kTrunkEB; ++e) acc[e] = bias;
    for (int c = 0; c < kMid; c += 4) {
      const float w0 = W2T[(c + 0) * kMid + t], w1 = W2T[(c + 1) * kMid + t];
      const float w2 = W2T[(c + 2) * kMid + t], w3 = W2T[(c + 3) * kMid + t];
#pragma unroll
      for (int e = 0; e < kTrunkEB; ++e) {
        const float4 a = *reinterpret_cast<const float4*>(&h[e][c]);
        acc[e] = fmaf(a.x, w0, acc[e]);
        acc[e] = fmaf(a.y, w1, acc[e]);
        acc[e] = fmaf(a.z, w2, acc[e]);
        acc[e] = fmaf(a.w, w3, acc[e]);
      }
    }
    __syncthreads();
#pragma unroll
    for (int e = 0; e < kTrunkEB; ++e) h[e][t] = acc[e];
  }
  __syncthreads();
  ln_gelu_rows(h, ne, ln2w, ln2b);
  __syncthreads();
  float* og = out_g + ((size_t)pair * E + e0) * kMid;
  for (int e = 0; e < ne; ++e) og[(size_t)e * kMid + t] = h[e][t];
}

// Trunk + low-rank radial coordinates (DESIGN.md 4.2): the same trunk, followed in the same CTA by
//   U[e, 0..r-1] = (g[e,:] - gmean) V[:, 0..r-1],   U[e, r] = 1 (bias slot),   U[e, r+1..63] = 0
// with the pair's cached centre gmean [128] and orthonormal basis V [128, 64] (columns >= r are zero), and by the check of that
// affine model on the edges of THIS forward: stats[pair] = (max |g - gmean - U V^T|, max |g|) accumulated with atomicMax (non-negative floats order like their bit
// patterns), read by the host once per forward.  g itself is only written when out_g != NULL.
constexpr int kVPad = 65;

__global__ void __launch_bounds__(128)
radial_trunk_u_kernel(const float* __restrict__ feat, int64_t E, int in_dim, const float* __restrict__ params, int64_t param_stride,
                      const float* __restrict__ Vall, const float* __restrict__ gmean, const int* __restrict__ ones_col,
                      float* __restrict__ out_g, float* __restrict__ out_U, float* __restrict__ stats) {
  extern __shared__ __align__(16) float dsm[];
  float (*h)[kMid + 4] = reinterpret_cast<float (*)[kMid + 4]>(dsm);                    // [32][132]
  float (*fs)[64] = reinterpret_cast<float (*)[64]>(dsm + kTrunkEB * (kMid + 4));       // [32][64]; reused for U
  float* Vs = dsm + kTrunkEB * (kMid + 4) + kTrunkEB * 64;                               // [128][65]
  const int pair = blockIdx.y;
  const int64_t e0 = (int64_t)blockIdx.x * kTrunkEB;
  const int ne = (int)max((int64_t)0, min((int64_t)kTrunkEB, E - e0));
  const int t = threadIdx.x;
  const float* P = params + (size_t)pair * param_stride;
  const float* W1T = P;
  const float* b1 = W1T + (size_t)in_dim * kMid;
  const float* ln1w = b1 + kMid;
  const float* ln1b = ln1w + kMid;
  const float* W2T = ln1b + kMid;
  const float* b2 = W2T + kMid * kMid;
  const float* ln2w = b2 + kMid;
  const float* ln2b = ln2w + kMid;
  const int rcol = ones_col[pair];                 // r: the bias slot; the basis has r columns

  for (int idx = t; idx < ne * in_dim; idx += 128) fs[idx / in_dim][idx % in_dim] = feat[(e0 + idx / in_dim) * in_dim + idx % in_dim];
  for (int idx = t; idx < kMid * 64; idx += 128) Vs[(idx >> 6) * kVPad + (idx & 63)] = Vall[(size_t)pair * kMid * 64 + idx];
  __syncthreads();
  {
    float acc[kTrunkEB];
    const float bias = b1[t];
#pragma unroll
    for (int e = 0; e < kTrunkEB; ++e) acc[e] = bias;
    for (int d = 0; d < in_dim; ++d) {
      const float w = W1T[d * kMid + t];
#pragma unroll
      for (int e = 0; e < kTrunkEB; ++e) acc[e] = fmaf(fs[e][d], w, acc[e]);
    }
#pragma unroll
    for (int e = 0; e < kTrunkEB; ++e) h[e][t] = acc[e];
  }
  __syncthreads();
  ln_gelu_rows(h, ne, ln1w, ln1b);
  __syncthreads();
  {
    float acc[kTrunkEB];
    const float bias = b2[t];
#pragma unroll
    for (int e = 0; e < kTrunkEB; ++e) acc[e] = bias;
    for (int c = 0; c < kMid; c += 4) {
      const float w0 = W2T[(c + 0) * kMid + t], w1 = W2T[(c + 1) * kMid + t];
      const float w2 = W2T[(c + 2) * kMid + t], w3 = W2T[(c + 3) * kMid + t];
#pragma unroll
      for (int e = 0; e < kTrunkEB; ++e) {
        const float4 a = *reinterpret_cast<const float4*>(&h[e][c]);
        acc[e] = fmaf(a.x, w0, acc[e]);
        acc[e] = fmaf(a.y, w1, acc[e]);
        acc[e] = fmaf(a.z, w2, acc[e]);
        acc[e] = fmaf(a.w, w3, acc[e]);
      }
    }
    __syncthreads();
#pragma unroll
    for (int e = 0; e < kTrunkEB; ++e) h[e][t] = acc[e];
  }
  __syncthreads();
  ln_gelu_rows(h, ne, ln2w, ln2b);
  __syncthreads();
  if (out_g != nullptr) {
    float* og = out_g + ((size_t)pair * E + e0) * kMid;
    for (int e = 0; e < ne; ++e) og[(size_t)e * kMid + t] = h[e][t];
  }
  // centre: the low-rank model is affine, g ~= gmean + U V^T (W3 gmean rides in the bias column of F'); max |g| before centring
  float gmax = 0.f;
  {
    const float mu = gmean[(size_t)pair * kMid + t];
    for (int e = 0; e < ne; ++e) {
      const float gv = h[e][t];
      gmax = fmaxf(gmax, fabsf(gv));
      h[e][t] = gv - mu;
    }
  }
  __syncthreads();
  // U = (g - gmean) V: thread t -> column k = t % 64 for 16 of the 32 edges
  {
    const int k = t & 63, eh = (t >> 6) * 16;
    float acc[16];
#pragma unroll
    for (int e = 0; e < 16; ++e) acc[e] = 0.f;
    if (k < rcol) {
      for (int j = 0; j < kMid; ++j) {
        const float v = Vs[j * kVPad + k];
#pragma unroll
        for (int e = 0; e < 16; ++e) acc[e] = fmaf(h[eh + e][j], v, acc[e]);
      }
    }
#pragma unroll
    for (int e = 0; e < 16; ++e) fs[eh + e][k] = acc[e];
  }
  __syncthreads();
  // residual of the cached basis on these edges: thread t = hidden unit
  float rmax = 0.f;
  if (rcol <= 32) {
    // this thread's row of V in registers; U rows are read as broadcast float4
    float vr[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) vr[k] = (k < rcol) ? Vs[t * kVPad + k] : 0.f;
    const int k4 = (rcol + 3) >> 2;
    for (int e = 0; e < ne; ++e) {
      float rec = 0.f;
      const float4* ur = reinterpret_cast<const float4*>(&fs[e][0]);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        if (q < k4) {
          const float4 u = ur[q];
          rec = fmaf(u.x, vr[4 * q], rec);
          rec = fmaf(u.y, vr[4 * q + 1], rec);
          rec = fmaf(u.z, vr[4 * q + 2], rec);
          rec = fmaf(u.w, vr[4 * q + 3], rec);
        }
      }
      rmax = fmaxf(rmax, fabsf(h[e][t] - rec));
    }
  } else {
    for (int e = 0; e < ne; ++e) {
      float rec = 0.f;
      for (int k = 0; k < rcol; ++k) rec = fmaf(fs[e][k], Vs[t * kVPad + k], rec);
      rmax = fmaxf(rmax, fabsf(h[e][t] - rec));
    }
  }
  rmax = warp_max(rmax);
  gmax = warp_max(gmax);
  if ((t & 31) == 0) {
    atomicMax(reinterpret_cast<unsigned int*>(stats + 2 * pair), __float_as_uint(rmax));
    atomicMax(reinterpret_cast<unsigned int*>(stats + 2 * pair + 1), __float_as_uint(gmax));
  }
  float* ou = out_U + ((size_t)pair * E + e0) * 64;
  for (int idx = t; idx < ne * 64; idx += 128) {
    const int e = idx >> 6, k = idx & 63;
    ou[idx] = (k == rcol) ? 1.f : fs[e][k];
  }
}

// Radial coordinates by table lookup (distance-only radial functions).  U(d) = (g(d) - gmean) V is a smooth curve in the ONE
// scalar the radial MLP sees, so the plan tabulates it in float64 on a uniform grid of [0, D] (the same samples the low-rank
// basis is computed from) and every forward interpolates: 4-point Lagrange (cubic, error ~ 0.023 h^4 |U''''|, checked against
// float64 at the grid midpoints when the table is built), 4 x KT loads + 4 x KT FMAs per (edge, pair) instead of the 41 kFLOP
// of the MLP.  Distances outside [0, D] (or non-finite) raise the pair's flag stats[pair] = (1, 1): the plan does not cover them.
__global__ void __launch_bounds__(256)
radial_table_kernel(const float* __restrict__ dist, int64_t E, const float* __restrict__ tab, int G, int KT, float inv_h, float Dmax,
                    const int* __restrict__ ones_col, int num_pairs, float* __restrict__ out_U, float* __restrict__ stats) {
  const int kq = KT / 4;                                       // float4 groups per table row
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int pair = blockIdx.y;
  if (idx >= E * 16) return;
  const int64_t e = idx >> 4;
  const int q = (int)(idx & 15);                               // float4 group of the 64-column output row
  const float d = dist[e];
  const bool ok = d >= 0.f && d <= Dmax;                       // (false for NaN)
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (q < kq) {
    const float t = fminf(fmaxf(ok ? d * inv_h : 0.f, 0.f), (float)(G - 1));
    int i0 = (int)floorf(t);
    i0 = max(1, min(i0, G - 3));
    const float f = t - (float)i0;                             // in [-1, 2]: nodes i0-1, i0, i0+1, i0+2 at -1, 0, 1, 2
    const float w0 = -f * (f - 1.f) * (f - 2.f) * (1.f / 6.f);
    const float w1 = (f + 1.f) * (f - 1.f) * (f - 2.f) * 0.5f;
    const float w2 = -(f + 1.f) * f * (f - 2.f) * 0.5f;
    const float w3 = (f + 1.f) * f * (f - 1.f) * (1.f / 6.f);
    const float4* row = reinterpret_cast<const float4*>(tab + ((size_t)pair * G + (i0 - 1)) * KT) + q;
    const float4 a = __ldg(row), b = __ldg(row + kq), c = __ldg(row + 2 * kq), dd = __ldg(row + 3 * kq);
    v.x = w0 * a.x + w1 * b.x + w2 * c.x + w3 * dd.x;
    v.y = w0 * a.y + w1 * b.y + w2 * c.y + w3 * dd.y;
    v.z = w0 * a.z + w1 * b.z + w2 * c.z + w3 * dd.z;
    v.w = w0 * a.w + w1 * b.w + w2 * c.w + w3 * dd.w;
  }
  const int oc = ones_col[pair];                               // bias slot
  if (oc >> 2 == q) {
    const int r = oc & 3;
    if (r == 0) v.x = 1.f; else if (r == 1) v.y = 1.f; else if (r == 2) v.z = 1.f; else v.w = 1.f;
  }
  reinterpret_cast<float4*>(out_U + ((size_t)pair * E + e) * 64)[q] = v;
  if (!ok && q == 0) {
    atomicMax(reinterpret_cast<unsigned int*>(stats + 2 * pair), __float_as_uint(1.f));
    atomicMax(reinterpret_cast<unsigned int*>(stats + 2 * pair + 1), __float_as_uint(1.f));
  }
}

}  // namespace se3

extern "C" int se3_radial_table_fwd(const float* dist, int64_t E, const float* table, int G, int KT, float Dmax, const int* ones_col,
                                    int num_pairs, float* out_U, float* stats, void* stream) {
  using namespace se3;
  SE3_REQUIRE(E > 0 && num_pairs > 0 && G >= 8 && Dmax > 0.f, "se3_radial_table_fwd: bad sizes");
  SE3_REQUIRE(KT >= 4 && KT <= 64 && KT % 4 == 0, "se3_radial_table_fwd: KT=%d must be a multiple of 4, <= 64", KT);
  SE3_REQUIRE(dist != nullptr && table != nullptr && ones_col != nullptr && out_U != nullptr && stats != nullptr, "se3_radial_table_fwd: null pointer");
  dim3 grid((unsigned)ceil_div(E * 16, 256), (unsigned)num_pairs);
  radial_table_kernel<<<grid, 256, 0, as_stream(stream)>>>(dist, E, table, G, KT, (float)((double)(G - 1) / (double)Dmax), Dmax, ones_col,
                                                          num_pairs, out_U, stats);
  SE3_LAUNCH_OK();
  return SE3_OK;
}

extern "C" int se3_radial_trunk_u_fwd(const float* feat, int64_t E, int in_dim, int num_pairs, const float* params, const float* V,
                                      const float* gmean, const int* ones_col, float* out_g, float* out_U, float* stats, void* stream) {
  using namespace se3;
  SE3_REQUIRE(E > 0 && num_pairs > 0, "se3_radial_trunk_u_fwd: bad sizes");
  SE3_REQUIRE(in_dim >= 1 && in_dim <= 64, "se3_radial_trunk_u_fwd: in_dim %d unsupported (1..64)", in_dim);
  SE3_REQUIRE(V != nullptr && gmean != nullptr && ones_col != nullptr && out_U != nullptr && stats != nullptr, "se3_radial_trunk_u_fwd: null pointer");
  const int64_t param_stride = (int64_t)in_dim * kMid + 3 * kMid + kMid * kMid + 3 * kMid;
  const size_t smem = sizeof(float) * (kTrunkEB * (kMid + 4) + kTrunkEB * 64 + kMid * kVPad);
  SE3_CUDA_OK(cudaFuncSetAttribute(radial_trunk_u_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid((unsigned)ceil_div(E, kTrunkEB), (unsigned)num_pairs);
  radial_trunk_u_kernel<<<grid, 128, smem, as_stream(stream)>>>(feat, E, in_dim, params, param_stride, V, gmean, ones_col, out_g, out_U, stats);
  SE3_LAUNCH_OK();
  return SE3_OK;
}

extern "C" int se3_radial_trunk_fwd(const float* feat, int64_t E, int in_dim, int num_pairs, const float* params,
                                    float* out_g, void* stream) {
  using namespace se3;
  SE3_REQUIRE(E > 0 && num_pairs > 0, "se3_radial_trunk_fwd: bad sizes");
  SE3_REQUIRE(in_dim >= 1 && in_dim <= 64, "se3_radial_trunk_fwd: in_dim %d unsupported (1..64)", in_dim);
  SE3_REQUIRE(out_g != nullptr, "se3_radial_trunk_fwd: no output buffer");
  const int64_t param_stride = (int64_t)in_dim * kMid + 3 * kMid + kMid * kMid + 3 * kMid;
  dim3 grid((unsigned)ceil_div(E, kTrunkEB), (unsigned)num_pairs);
  radial_trunk_kernel<<<grid, 128, 0, as_stream(stream)>>>(feat, E, in_dim, params, param_stride, out_g);
  SE3_LAUNCH_OK();
  return SE3_OK;
}
