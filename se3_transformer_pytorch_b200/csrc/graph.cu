// K1: neighbour graph, pair-feature gather and masked-mean pooling.
//
// Replaces the dense [b,n,n-1] temporaries + torch.topk + batched_index_select of the reference
// (se3_transformer_pytorch.py:1171-1294, utils.py:56-80) with one CTA per query node that keeps the whole
// distance row in shared memory, sorts (distance, column) keys bitonically and emits only the k winners.  The same row body
// serves padded batches [b, n] (knn_kernel) and packed batches of clouds of different sizes (knn_varlen_kernel).
#include "common.cuh"
#include <cfloat>
#include <vector>

namespace se3 {

__host__ __device__ inline int knn_npad(int n) {
  int npad = 2;
  while (npad < n - 1) npad <<= 1;
  return npad;
}

// The neighbour list of node i of one cloud of n nodes (c = that cloud's coordinates, [n, 3]); shared by the padded
// (knn_kernel) and the packed (knn_varlen_kernel) search so that both produce the same bits.
// key = (bits(modified distance) << 32) | column on the self-removed grid.  Distances are >= 0 so the IEEE bit pattern is
// order preserving; equal distances order by column, which is the stable-argsort tie rule the oracle uses (torch.topk
// leaves ties unspecified).  nbr_row / adj_row: row i of the cloud's [n, n] pair masks (or NULL); node_mask: the cloud's
// [n] node mask (or NULL).  Writes slots [0, K_out) of the row at out_*; slots r >= k are copies of slot k - 1 with mask 0,
// and indices are offset by j_base.
template <int THREADS>
__device__ __forceinline__ void knn_row(unsigned long long* keys, const float* __restrict__ c, int n, int i, int k, int npad,
                                        const uint8_t* __restrict__ nbr_row, const uint8_t* __restrict__ adj_row,
                                        const uint8_t* __restrict__ node_mask, float valid_radius, int causal, int K_out,
                                        int64_t j_base, int64_t* __restrict__ out_idx, uint8_t* __restrict__ out_mask,
                                        float* __restrict__ out_rel_pos, float* __restrict__ out_rel_dist) {
  const float xi = c[i * 3 + 0], yi = c[i * 3 + 1], zi = c[i * 3 + 2];
  for (int jc = threadIdx.x; jc < npad; jc += THREADS) {
    unsigned long long key = ~0ull;
    if (jc < n - 1) {
      const int j = jc + (jc >= i);
      const float dx = xi - c[j * 3 + 0], dy = yi - c[j * 3 + 1], dz = zi - c[j * 3 + 2];
      float d = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
      if (nbr_row && !nbr_row[j]) d = FLT_MAX;
      if (adj_row && adj_row[j]) d = 0.f;
      if (causal && jc >= i) d = FLT_MAX;
      key = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)jc;
    }
    keys[jc] = key;
  }
  __syncthreads();
  // bitonic sort, ascending
  for (int size = 2; size <= npad; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = threadIdx.x; t < (npad >> 1); t += THREADS) {
        const int lo = 2 * t - (t & (stride - 1));
        const int hi = lo + stride;
        const bool up = ((lo & size) == 0);
        const unsigned long long a = keys[lo], bb = keys[hi];
        if ((a > bb) == up) { keys[lo] = bb; keys[hi] = a; }
      }
      __syncthreads();
    }
  }
  const bool mi = node_mask ? node_mask[i] != 0 : true;
  for (int r = threadIdx.x; r < K_out; r += THREADS) {
    const unsigned long long key = keys[r < k ? r : k - 1];
    const int jc = (int)(key & 0xffffffffu);
    const float dmod = __uint_as_float((unsigned)(key >> 32));
    const int j = jc + (jc >= i);
    const float dx = xi - c[j * 3 + 0], dy = yi - c[j * 3 + 1], dz = zi - c[j * 3 + 2];
    const float d = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
    bool m = r < k && dmod <= valid_radius;
    if (node_mask) m = m && mi && node_mask[j] != 0;
    out_idx[r] = j_base + j;
    out_mask[r] = m ? 1 : 0;
    out_rel_pos[r * 3 + 0] = dx;
    out_rel_pos[r * 3 + 1] = dy;
    out_rel_pos[r * 3 + 2] = dz;
    out_rel_dist[r] = d;
  }
}

// One CTA per (cloud, node i) of a padded batch [b, n].
template <int THREADS>
__global__ void __launch_bounds__(THREADS)
knn_kernel(const float* __restrict__ coors, const uint8_t* __restrict__ node_mask,
           const uint8_t* __restrict__ neighbor_mask, const uint8_t* __restrict__ sparse_adj,
           int n, int k, int npad, float valid_radius, int causal,
           int64_t* __restrict__ out_idx, uint8_t* __restrict__ out_mask,
           float* __restrict__ out_rel_pos, float* __restrict__ out_rel_dist) {
  extern __shared__ unsigned long long keys[];
  const int i = blockIdx.x, b = blockIdx.y;
  const size_t row = ((size_t)b * n + i) * n;
  const size_t o = ((size_t)b * n + i) * k;
  knn_row<THREADS>(keys, coors + (size_t)b * n * 3, n, i, k, npad, neighbor_mask ? neighbor_mask + row : nullptr,
                   sparse_adj ? sparse_adj + row : nullptr, node_mask ? node_mask + (size_t)b * n : nullptr, valid_radius, causal,
                   k, 0, out_idx + o, out_mask + o, out_rel_pos + o * 3, out_rel_dist + o);
}

// One CTA per node of a packed batch: clouds c of n_c = cu_seqlens[c+1] - cu_seqlens[c] nodes laid end to end.  The CTA finds
// its cloud by binary search, searches that cloud only (local columns, the cloud's own k_c) and writes K >= k_c slots with
// global indices.  Pair masks are the clouds' [n_c, n_c] matrices flattened end to end, cloud c starting at pair_off[c].
template <int THREADS>
__global__ void __launch_bounds__(THREADS)
knn_varlen_kernel(const float* __restrict__ coors, const int64_t* __restrict__ cu_seqlens, const int* __restrict__ k_per_cloud,
                  const uint8_t* __restrict__ neighbor_mask, const uint8_t* __restrict__ sparse_adj,
                  const int64_t* __restrict__ pair_off, int num_clouds, int K, float valid_radius, int causal,
                  int64_t* __restrict__ out_idx, uint8_t* __restrict__ out_mask,
                  float* __restrict__ out_rel_pos, float* __restrict__ out_rel_dist) {
  extern __shared__ unsigned long long keys[];
  const int64_t t = blockIdx.x;
  int lo = 0, hi = num_clouds - 1;               // the last cloud c with cu_seqlens[c] <= t
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (cu_seqlens[mid] <= t) lo = mid; else hi = mid - 1;
  }
  const int64_t start = cu_seqlens[lo];
  const int n = (int)(cu_seqlens[lo + 1] - start), i = (int)(t - start);
  const size_t row = neighbor_mask || sparse_adj ? (size_t)pair_off[lo] + (size_t)i * n : 0;
  const size_t o = (size_t)t * K;
  knn_row<THREADS>(keys, coors + start * 3, n, i, k_per_cloud[lo], knn_npad(n), neighbor_mask ? neighbor_mask + row : nullptr,
                   sparse_adj ? sparse_adj + row : nullptr, nullptr, valid_radius, causal, K, start, out_idx + o, out_mask + o,
                   out_rel_pos + o * 3, out_rel_dist + o);
}

__global__ void gather_pairs_kernel(const float* __restrict__ pf, const int64_t* __restrict__ idx, int n, int k, int e,
                                    int64_t total, float* __restrict__ out) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int c = (int)(t % e);
  const int64_t edge = t / e;               // (b*n + i)*k + kk
  const int64_t bi = edge / k;              // b*n + i
  const int64_t j = idx[edge];
  out[t] = pf[(bi * n + j) * e + c];
}

// x [B,K,C] -> out [B,C]; masked_mean semantics of utils.py:72-80.
__global__ void pool_kernel(const float* __restrict__ x, const uint8_t* __restrict__ mask, int K, int64_t C,
                            float* __restrict__ out) {
  const int64_t bidx = blockIdx.x;
  float cnt = 0.f;
  if (mask) {
    for (int kk = 0; kk < K; ++kk) cnt += mask[bidx * K + kk] ? 1.f : 0.f;
  } else {
    cnt = (float)K;
  }
  for (int64_t c = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; c < C; c += (int64_t)gridDim.y * blockDim.x) {
    float s = 0.f;
    for (int kk = 0; kk < K; ++kk) {
      if (!mask || mask[bidx * K + kk]) s += x[(bidx * K + kk) * C + c];
    }
    out[bidx * C + c] = cnt > 0.f ? s / cnt : 0.f;
  }
}

}  // namespace se3

extern "C" int se3_knn_fwd(const float* coors, const uint8_t* node_mask, const uint8_t* neighbor_mask,
                           const uint8_t* sparse_adj, int b, int n, int k, float valid_radius, int causal,
                           int64_t* out_idx, uint8_t* out_mask, float* out_rel_pos, float* out_rel_dist, void* stream) {
  using namespace se3;
  SE3_REQUIRE(b > 0 && n > 1, "se3_knn_fwd: need b > 0 and n > 1 (got b=%d n=%d)", b, n);
  SE3_REQUIRE(k >= 1 && k <= n - 1, "se3_knn_fwd: k must be in [1, n-1] (got k=%d n=%d)", k, n);
  SE3_REQUIRE(n - 1 <= 4096, "se3_knn_fwd: n-1 = %d exceeds the 4096-column shared-memory sort", n - 1);
  const int npad = knn_npad(n);
  constexpr int THREADS = 256;
  dim3 grid(n, b);
  const size_t smem = (size_t)npad * sizeof(unsigned long long);
  knn_kernel<THREADS><<<grid, THREADS, smem, as_stream(stream)>>>(coors, node_mask, neighbor_mask, sparse_adj, n, k, npad,
                                                                  valid_radius, causal, out_idx, out_mask, out_rel_pos,
                                                                  out_rel_dist);
  SE3_LAUNCH_OK();
  return SE3_OK;
}

extern "C" int se3_knn_varlen_fwd(const float* coors, const int64_t* cu_seqlens, const int* k_per_cloud,
                                  const uint8_t* neighbor_mask, const uint8_t* sparse_adj, const int64_t* pair_off, int num_clouds,
                                  int64_t total, int K, int max_len, float valid_radius, int causal, int64_t* out_idx,
                                  uint8_t* out_mask, float* out_rel_pos, float* out_rel_dist, void* stream) {
  using namespace se3;
  SE3_REQUIRE(num_clouds > 0 && total > 0 && K > 0, "se3_knn_varlen_fwd: need num_clouds, total, K > 0 (got %d, %lld, %d)",
              num_clouds, (long long)total, K);
  SE3_REQUIRE(total < (1ll << 31), "se3_knn_varlen_fwd: %lld nodes exceed the 1-D grid", (long long)total);
  SE3_REQUIRE(max_len >= 2 && max_len - 1 <= 4096, "se3_knn_varlen_fwd: max_len = %d must be in [2, 4097]", max_len);
  // the sizes live on the device: read them back once (a few hundred bytes) so that a bad batch is refused, not read out of bounds
  std::vector<int64_t> cu(num_clouds + 1), off(num_clouds);
  std::vector<int> kc(num_clouds);
  cudaStream_t s = as_stream(stream);
  SE3_CUDA_OK(cudaMemcpyAsync(cu.data(), cu_seqlens, cu.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  SE3_CUDA_OK(cudaMemcpyAsync(kc.data(), k_per_cloud, kc.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
  const bool pairs = neighbor_mask || sparse_adj;
  if (pairs) SE3_CUDA_OK(cudaMemcpyAsync(off.data(), pair_off, off.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
  SE3_CUDA_OK(cudaStreamSynchronize(s));
  SE3_REQUIRE(cu[0] == 0 && cu[num_clouds] == total, "se3_knn_varlen_fwd: cu_seqlens must run from 0 to total = %lld (got %lld .. %lld)",
              (long long)total, (long long)cu[0], (long long)cu[num_clouds]);
  int64_t pairs_before = 0;
  for (int c = 0; c < num_clouds; ++c) {
    const int64_t n = cu[c + 1] - cu[c];
    SE3_REQUIRE(n >= 2 && n - 1 <= 4096, "se3_knn_varlen_fwd: cloud %d has %lld nodes; each cloud needs 2 .. 4097", c, (long long)n);
    SE3_REQUIRE(n <= max_len, "se3_knn_varlen_fwd: cloud %d has %lld nodes > max_len = %d", c, (long long)n, max_len);
    SE3_REQUIRE(kc[c] >= 1 && kc[c] <= n - 1, "se3_knn_varlen_fwd: k of cloud %d must be in [1, n_c - 1] (got k=%d n_c=%lld)", c,
                kc[c], (long long)n);
    SE3_REQUIRE(kc[c] <= K, "se3_knn_varlen_fwd: K = %d is smaller than k = %d of cloud %d", K, kc[c], c);
    SE3_REQUIRE(!pairs || off[c] == pairs_before, "se3_knn_varlen_fwd: pair_off[%d] = %lld, expected sum of n_c^2 before it = %lld", c,
                (long long)off[c], (long long)pairs_before);
    pairs_before += n * n;
  }
  constexpr int THREADS = 256;
  const size_t smem = (size_t)knn_npad(max_len) * sizeof(unsigned long long);
  knn_varlen_kernel<THREADS><<<(unsigned)total, THREADS, smem, s>>>(coors, cu_seqlens, k_per_cloud, neighbor_mask, sparse_adj,
                                                                     pair_off, num_clouds, K, valid_radius, causal, out_idx,
                                                                     out_mask, out_rel_pos, out_rel_dist);
  SE3_LAUNCH_OK();
  return SE3_OK;
}

extern "C" int se3_gather_pairs_fwd(const float* pair_feat, const int64_t* idx, int b, int n, int k, int e, float* out,
                                    void* stream) {
  using namespace se3;
  SE3_REQUIRE(b > 0 && n > 0 && k > 0 && e > 0, "se3_gather_pairs_fwd: bad sizes");
  const int64_t total = (int64_t)b * n * k * e;
  const int threads = 256;
  gather_pairs_kernel<<<(unsigned)ceil_div(total, threads), threads, 0, as_stream(stream)>>>(pair_feat, idx, n, k, e, total, out);
  SE3_LAUNCH_OK();
  return SE3_OK;
}

extern "C" int se3_pool_fwd(const float* x, const uint8_t* mask, int64_t B, int K, int64_t C, float* out, void* stream) {
  using namespace se3;
  SE3_REQUIRE(B > 0 && K > 0 && C > 0, "se3_pool_fwd: bad sizes");
  SE3_REQUIRE(B < (1ll << 31), "se3_pool_fwd: B too large");
  const int threads = 256;
  dim3 grid((unsigned)B, (unsigned)std::min<int64_t>(ceil_div(C, threads), 64));
  pool_kernel<<<grid, threads, 0, as_stream(stream)>>>(x, mask, K, C, out);
  SE3_LAUNCH_OK();
  return SE3_OK;
}
