// K5: per-degree attention over the neighbour list (AttentionSE3.forward, se3_transformer_pytorch.py:476-517;
// OneHeadedKVAttentionSE3, S:612-652).  One warp per (node, head): lanes stride over the contiguous
// (dim_head x 2l+1) slice of a key/value, warp-shuffle reductions give the logits, softmax is done redundantly in
// every lane, and keys/values are read exactly once with coalesced loads.  HBM-bound by design.
#include "common.cuh"
#include <cfloat>

namespace se3 {

constexpr int kAttnWarps = 4;

struct AttnArgs {
  const float* q; const float* k; const float* v; const int64_t* k_idx;
  const float* self_k; const float* self_v; const float* null_k; const float* null_v;
  const float* global_k; const float* global_v; const uint8_t* nmask;
  float* out;
  int b, n, K, H, Dh, M, kv_heads, G, has_null, has_self;
  float scale;
};

// pointer to the [Dh*M] slice of key/value number j (in the concatenated order) for node (b,i), kv head hk
__device__ __forceinline__ const float* kv_ptr(const AttnArgs& a, bool is_key, int64_t bb, int64_t i, int j, int hk, int L, int Ckv) {
  const size_t hoff = (size_t)hk * L;
  const size_t slab = (size_t)Ckv * a.M;
  if (j < a.G) return (is_key ? a.global_k : a.global_v) + ((size_t)bb * a.G + j) * slab + hoff;
  j -= a.G;
  if (a.has_null) { if (j == 0) return (is_key ? a.null_k : a.null_v) + hoff; j -= 1; }
  if (a.has_self) { if (j == 0) return (is_key ? a.self_k : a.self_v) + ((size_t)bb * a.n + i) * slab + hoff; j -= 1; }
  if (is_key && a.k_idx) return a.k + ((size_t)bb * a.n + a.k_idx[((size_t)bb * a.n + i) * a.K + j]) * slab + hoff;
  return (is_key ? a.k : a.v) + (((size_t)bb * a.n + i) * a.K + j) * slab + hoff;
}

template <int NL>   // NL = ceil(L / 32) register slots per lane
__global__ void __launch_bounds__(kAttnWarps * 32)
attn_kernel(AttnArgs a) {
  extern __shared__ float logits_all[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t node = (int64_t)blockIdx.x;                 // b*n + i
  const int h = blockIdx.y * kAttnWarps + warp;
  if (h >= a.H) return;
  const int64_t bb = node / a.n, i = node % a.n;
  const int L = a.Dh * a.M;
  const int Ckv = a.kv_heads * a.Dh;
  const int hk = a.kv_heads == 1 ? 0 : h;
  const int prefix = a.G + a.has_null + a.has_self;
  const int J = prefix + a.K;
  float* logits = logits_all + (size_t)warp * J;

  float qv[NL];
  const float* qp = a.q + ((size_t)node * a.H + h) * L;
#pragma unroll
  for (int t = 0; t < NL; ++t) { const int l = lane + 32 * t; qv[t] = l < L ? qp[l] : 0.f; }

  // logits, two keys in flight
  for (int j = 0; j < J; j += 2) {
    const float* k0 = kv_ptr(a, true, bb, i, j, hk, L, Ckv);
    const bool has1 = (j + 1 < J);
    const float* k1 = has1 ? kv_ptr(a, true, bb, i, j + 1, hk, L, Ckv) : k0;
    float s0 = 0.f, s1 = 0.f;
#pragma unroll
    for (int t = 0; t < NL; ++t) {
      const int l = lane + 32 * t;
      if (l < L) { s0 = fmaf(qv[t], k0[l], s0); s1 = fmaf(qv[t], k1[l], s1); }
    }
    s0 = warp_sum(s0) * a.scale;
    s1 = warp_sum(s1) * a.scale;
    if (a.nmask) {
      const uint8_t* mrow = a.nmask + (size_t)node * a.K;
      if (j >= prefix && !mrow[j - prefix]) s0 = -FLT_MAX;
      if (has1 && j + 1 >= prefix && !mrow[j + 1 - prefix]) s1 = -FLT_MAX;
    }
    if (lane == 0) { logits[j] = s0; if (has1) logits[j + 1] = s1; }
  }
  __syncwarp();
  float mx = -FLT_MAX;
  for (int j = lane; j < J; j += 32) mx = fmaxf(mx, logits[j]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j < J; j += 32) { const float ex = expf(logits[j] - mx); logits[j] = ex; sum += ex; }
  sum = warp_sum(sum);
  __syncwarp();
  const float inv = 1.f / sum;

  float acc[NL];
#pragma unroll
  for (int t = 0; t < NL; ++t) acc[t] = 0.f;
  for (int j = 0; j < J; j += 2) {
    const float* v0 = kv_ptr(a, false, bb, i, j, hk, L, Ckv);
    const bool has1 = (j + 1 < J);
    const float* v1 = has1 ? kv_ptr(a, false, bb, i, j + 1, hk, L, Ckv) : v0;
    const float a0 = logits[j] * inv;
    const float a1 = has1 ? logits[j + 1] * inv : 0.f;
#pragma unroll
    for (int t = 0; t < NL; ++t) {
      const int l = lane + 32 * t;
      if (l < L) { acc[t] = fmaf(a0, v0[l], acc[t]); acc[t] = fmaf(a1, v1[l], acc[t]); }
    }
  }
  float* op = a.out + ((size_t)node * a.H + h) * L;
#pragma unroll
  for (int t = 0; t < NL; ++t) { const int l = lane + 32 * t; if (l < L) op[l] = acc[t]; }
}

// Attention over keys / values that are still in the EDGE-ALIGNED frame (DESIGN.md 4.5): kp, vp [E, P, Ckv] are the component-
// major outputs out' of se3_zgemm_fwd and D [E, P, P] the Wigner matrices of the edge frames, k[e,d,:] = D(e) kp[e,:,d].  The
// rotation back to the global frame (S:237-254 re-associated) happens here, on the fly: the query is rotated INTO the frame of
// every edge for the logit (sum_{d,m} q k = sum_{d,n} (D^T q)[d,n] kp[n,d]) and every value is rotated out before it is
// accumulated, so the global-frame K / V tensors are never written or read.  Prefix keys (global / null / self) are node level
// and already in the global frame.  One warp per (node, head); lanes over dim_head.  The D of the node's edges sit in shared
// memory: all K of them when K <= kAttnEdgeTile, else (kTiled) tiles of kAttnEdgeTile edges staged in turn by the whole block,
// so that only the logits grow with K.  In the tiled kernel a warp past the last head computes that head again and stores
// nothing, so that every warp reaches every block barrier.  kTiled is a template switch because block barriers inside the key
// loops cost registers.
constexpr int kAttnEdgeTile = 32;

// D of edges e0 .. e0 + te - 1 (at most K - e0) of this node into sD, by the whole block
template <int P>
__device__ __forceinline__ void stage_frames(float* sD, const float* __restrict__ Dmat, int64_t node, int K, int e0, int te, bool sync_before) {
  if (sync_before) __syncthreads();                           // every warp is done with the previous tile
  const int cnt = min(te, K - e0) * P * P;
  const float* src = Dmat + ((size_t)node * K + e0) * P * P;
  for (int t = threadIdx.x; t < cnt; t += blockDim.x) sD[t] = src[t];
  __syncthreads();
}

template <int P, int ND, bool kTiled>
__global__ void __launch_bounds__(kAttnWarps * 32)
attn_aligned_kernel(AttnArgs a, const float* __restrict__ Dmat, int k_aligned) {
  extern __shared__ float smem_dyn[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t node = (int64_t)blockIdx.x;
  const int h_warp = blockIdx.y * kAttnWarps + warp;
  const int h = min(h_warp, a.H - 1);
  const int64_t bb = node / a.n, i = node % a.n;
  const int Ckv = a.kv_heads * a.Dh;
  const int prefix = a.G + a.has_null + a.has_self;
  const int J = prefix + a.K;
  const int te = kTiled ? kAttnEdgeTile : a.K;
  float* sD = smem_dyn;                                       // [te][P*P]: D of edges t0 .. t0 + te - 1
  float* logits = smem_dyn + (size_t)te * P * P + (size_t)warp * J;
  if (!kTiled) {
    stage_frames<P>(sD, Dmat, node, a.K, 0, te, false);
    if (h_warp >= a.H) return;                                // no block barrier follows
  }
  const int hk = a.kv_heads == 1 ? 0 : h;
  const int L = a.Dh * P;

  float qv[ND][P];
#pragma unroll
  for (int t = 0; t < ND; ++t) {
    const int d = lane + 32 * t;
#pragma unroll
    for (int m = 0; m < P; ++m) qv[t][m] = (d < a.Dh) ? a.q[((size_t)node * a.H + h) * L + (size_t)d * P + m] : 0.f;
  }
  const uint8_t* mrow = a.nmask ? a.nmask + (size_t)node * a.K : nullptr;
  for (int j = 0, t0 = kTiled ? -te : 0; j < J; ++j) {
    const int jj = j - prefix;
    if (kTiled && k_aligned && jj == t0 + te) { t0 = jj; stage_frames<P>(sD, Dmat, node, a.K, t0, te, t0 > 0); }
    float s = 0.f;
    if (j < prefix || !k_aligned) {
      const float* kp = kv_ptr(a, true, bb, i, j, hk, L, Ckv);
#pragma unroll
      for (int t = 0; t < ND; ++t) {
        const int d = lane + 32 * t;
        if (d < a.Dh) {
#pragma unroll
          for (int m = 0; m < P; ++m) s = fmaf(qv[t][m], kp[(size_t)d * P + m], s);
        }
      }
    } else {
      if (mrow == nullptr || mrow[jj]) {
        const float* dm = sD + (jj - t0) * P * P;
        const float* kp = a.k + (((size_t)node * a.K + jj) * P) * Ckv + (size_t)hk * a.Dh;
#pragma unroll
        for (int t = 0; t < ND; ++t) {
          const int d = lane + 32 * t;
          if (d < a.Dh) {
#pragma unroll
            for (int n = 0; n < P; ++n) {
              float qn = 0.f;                                   // (D^T q)[d, n]
#pragma unroll
              for (int m = 0; m < P; ++m) qn = fmaf(dm[m * P + n], qv[t][m], qn);
              s = fmaf(qn, kp[(size_t)n * Ckv + d], s);
            }
          }
        }
      }
    }
    s = warp_sum(s) * a.scale;
    if (mrow && j >= prefix && !mrow[j - prefix]) s = -FLT_MAX;
    if (lane == 0) logits[j] = s;
  }
  __syncwarp();
  float mx = -FLT_MAX;
  for (int j = lane; j < J; j += 32) mx = fmaxf(mx, logits[j]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int j = lane; j < J; j += 32) { const float ex = expf(logits[j] - mx); logits[j] = ex; sum += ex; }
  sum = warp_sum(sum);
  __syncwarp();
  const float inv = 1.f / sum;

  float acc[ND][P];
#pragma unroll
  for (int t = 0; t < ND; ++t)
#pragma unroll
    for (int m = 0; m < P; ++m) acc[t][m] = 0.f;
  for (int j = 0, t0 = kTiled ? -te : 0; j < J; ++j) {
    const int jj = j - prefix;
    if (kTiled && jj == t0 + te) { t0 = jj; stage_frames<P>(sD, Dmat, node, a.K, t0, te, true); }
    const float aj = logits[j] * inv;
    if (j < prefix) {
      const float* vp = kv_ptr(a, false, bb, i, j, hk, L, Ckv);
#pragma unroll
      for (int t = 0; t < ND; ++t) {
        const int d = lane + 32 * t;
        if (d < a.Dh) {
#pragma unroll
          for (int m = 0; m < P; ++m) acc[t][m] = fmaf(aj, vp[(size_t)d * P + m], acc[t][m]);
        }
      }
    } else {
      if (aj == 0.f) continue;                                  // masked neighbour (warp uniform)
      const float* dm = sD + (jj - t0) * P * P;
      const float* vp = a.v + (((size_t)node * a.K + jj) * P) * Ckv + (size_t)hk * a.Dh;
#pragma unroll
      for (int t = 0; t < ND; ++t) {
        const int d = lane + 32 * t;
        if (d < a.Dh) {
          float vn[P];
#pragma unroll
          for (int n = 0; n < P; ++n) vn[n] = aj * vp[(size_t)n * Ckv + d];
#pragma unroll
          for (int m = 0; m < P; ++m) {
            float r = acc[t][m];
#pragma unroll
            for (int n = 0; n < P; ++n) r = fmaf(dm[m * P + n], vn[n], r);
            acc[t][m] = r;
          }
        }
      }
    }
  }
  if (h_warp >= a.H) return;
#pragma unroll
  for (int t = 0; t < ND; ++t) {
    const int d = lane + 32 * t;
    if (d < a.Dh) {
#pragma unroll
      for (int m = 0; m < P; ++m) a.out[((size_t)node * a.H + h) * L + (size_t)d * P + m] = acc[t][m];
    }
  }
}

template <int P>
static int launch_attn_aligned(const AttnArgs& a, const float* D, int k_aligned, cudaStream_t s) {
  const int J = a.G + a.has_null + a.has_self + a.K;
  const bool tiled = a.K > kAttnEdgeTile;
  const int te = tiled ? kAttnEdgeTile : a.K;
  const size_t smem = ((size_t)te * P * P + (size_t)kAttnWarps * J) * sizeof(float);
  SE3_REQUIRE(smem <= 200 * 1024, "se3_attn_aligned_fwd: %d keys per query exceed the shared-memory budget", J);
  dim3 grid((unsigned)((int64_t)a.b * a.n), (unsigned)ceil_div(a.H, kAttnWarps));
  const int warps = min(a.H, kAttnWarps);                     // (fewer than kAttnWarps heads: no idle warps)
  const int ND = (int)ceil_div(a.Dh, 32);
#define SE3_AA_T(NDV, TILED)                                                                                                 \
  {                                                                                                                          \
    if (smem > 48 * 1024) SE3_CUDA_OK(cudaFuncSetAttribute(attn_aligned_kernel<P, NDV, TILED>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    attn_aligned_kernel<P, NDV, TILED><<<grid, warps * 32, smem, s>>>(a, D, k_aligned);                                      \
  }
#define SE3_AA(NDV) { if (tiled) SE3_AA_T(NDV, true) else SE3_AA_T(NDV, false) }
  if (ND <= 1) SE3_AA(1) else if (ND <= 2) SE3_AA(2) else SE3_AA(4)
#undef SE3_AA_T
#undef SE3_AA
  SE3_LAUNCH_OK();
  return SE3_OK;
}

}  // namespace se3

extern "C" int se3_attn_aligned_fwd(const float* q, const float* k, const float* v, const float* D, int k_aligned, const int64_t* k_idx,
                                    const float* self_k, const float* self_v, const float* null_k, const float* null_v,
                                    const float* global_k, const float* global_v, int G, const uint8_t* nmask, int b, int n, int K, int H,
                                    int Dh, int M, int kv_heads, float scale, float* out, void* stream) {
  using namespace se3;
  SE3_REQUIRE(b > 0 && n > 0 && K > 0 && H > 0 && Dh > 0, "se3_attn_aligned_fwd: bad sizes");
  SE3_REQUIRE(M == 3 || M == 5 || M == 7 || M == 9 || M == 11, "se3_attn_aligned_fwd: M=%d (degrees 1..5 only; degree 0 needs no rotation)", M);
  SE3_REQUIRE(Dh <= 128, "se3_attn_aligned_fwd: dim_head=%d exceeds 128", Dh);
  SE3_REQUIRE(kv_heads == H || kv_heads == 1, "se3_attn_aligned_fwd: kv_heads must be H or 1");
  SE3_REQUIRE(D != nullptr, "se3_attn_aligned_fwd: D is required");
  SE3_REQUIRE((self_k == nullptr) == (self_v == nullptr) && (null_k == nullptr) == (null_v == nullptr), "se3_attn_aligned_fwd: k/v prefix mismatch");
  SE3_REQUIRE(G == 0 || (global_k && global_v), "se3_attn_aligned_fwd: G > 0 needs global_k/global_v");
  AttnArgs a{q, k, v, k_idx, self_k, self_v, null_k, null_v, global_k, global_v, nmask, out,
             b, n, K, H, Dh, M, kv_heads, G, null_k ? 1 : 0, self_k ? 1 : 0, scale};
  cudaStream_t s = as_stream(stream);
  switch (M) {
    case 3: return launch_attn_aligned<3>(a, D, k_aligned, s);
    case 5: return launch_attn_aligned<5>(a, D, k_aligned, s);
    case 7: return launch_attn_aligned<7>(a, D, k_aligned, s);
    case 9: return launch_attn_aligned<9>(a, D, k_aligned, s);
    default: return launch_attn_aligned<11>(a, D, k_aligned, s);
  }
}

extern "C" int se3_attn_fwd(const float* q, const float* k, const float* v, const int64_t* k_idx, const float* self_k,
                            const float* self_v, const float* null_k, const float* null_v, const float* global_k,
                            const float* global_v, int G, const uint8_t* nmask, int b, int n, int K, int H, int Dh, int M,
                            int kv_heads, float scale, float* out, void* stream) {
  using namespace se3;
  SE3_REQUIRE(b > 0 && n > 0 && K > 0 && H > 0 && Dh > 0 && M > 0, "se3_attn_fwd: bad sizes");
  SE3_REQUIRE(kv_heads == H || kv_heads == 1, "se3_attn_fwd: kv_heads must be H or 1");
  SE3_REQUIRE((self_k == nullptr) == (self_v == nullptr) && (null_k == nullptr) == (null_v == nullptr), "se3_attn_fwd: k/v prefix mismatch");
  SE3_REQUIRE(G == 0 || (global_k && global_v), "se3_attn_fwd: G > 0 needs global_k/global_v");
  const int L = Dh * M;
  SE3_REQUIRE(L <= 32 * 32, "se3_attn_fwd: dim_head*(2l+1) = %d exceeds 1024", L);
  AttnArgs a{q, k, v, k_idx, self_k, self_v, null_k, null_v, global_k, global_v, nmask, out,
             b, n, K, H, Dh, M, kv_heads, G, null_k ? 1 : 0, self_k ? 1 : 0, scale};
  const int J = G + a.has_null + a.has_self + K;
  const size_t smem = (size_t)kAttnWarps * J * sizeof(float);
  SE3_REQUIRE(smem <= 200 * 1024, "se3_attn_fwd: %d keys per query exceed the shared-memory logits buffer", J);
  dim3 grid((unsigned)((int64_t)b * n), (unsigned)ceil_div(H, kAttnWarps));
  cudaStream_t s = as_stream(stream);
  const int NL = (int)ceil_div(L, 32);
#define SE3_ATTN_CASE(N)                                                                                           \
  {                                                                                                                \
    if (smem > 48 * 1024) SE3_CUDA_OK(cudaFuncSetAttribute(attn_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
    attn_kernel<N><<<grid, kAttnWarps * 32, smem, s>>>(a);                                                         \
  }
  if (NL <= 1) SE3_ATTN_CASE(1)
  else if (NL <= 2) SE3_ATTN_CASE(2)
  else if (NL <= 4) SE3_ATTN_CASE(4)
  else if (NL <= 6) SE3_ATTN_CASE(6)
  else if (NL <= 8) SE3_ATTN_CASE(8)
  else if (NL <= 10) SE3_ATTN_CASE(10)
  else if (NL <= 14) SE3_ATTN_CASE(14)
  else if (NL <= 18) SE3_ATTN_CASE(18)
  else if (NL <= 22) SE3_ATTN_CASE(22)
  else SE3_ATTN_CASE(32)
#undef SE3_ATTN_CASE
  SE3_LAUNCH_OK();
  return SE3_OK;
}
