// Node digests for the prefix cache of the paged causal decoder (DESIGN.md 10.4, se3_prefix_keys_fwd).
//
// The digest of node i is two 64-bit lanes, each a wrapping sum over the node's input words of
//   mix64(word ^ mix64(seed_lane + (4 k + tag + 1) * G)),
// finished with mix64, where k is the word's index within its section and tag the section: 0 the conv_in input row (float32
// bits, degrees concatenated), 1 the coordinates (float32 bits), 2 the edges of columns j < i (int64 tokens, or float32 bits of
// the j * edge_dim + e-th value), 3 the neighbour mask of columns j < i (one byte each).  Integer sums do not depend on the order
// of reduction, so the digest is the same for any block size or thread mapping.
#include "common.cuh"

namespace se3 {
namespace {

constexpr uint64_t PREFIX_SEED0 = 0x243F6A8885A308D3ull;
constexpr uint64_t PREFIX_SEED1 = 0x13198A2E03707344ull;
constexpr uint64_t PREFIX_GOLD = 0x9E3779B97F4A7C15ull;
constexpr int PREFIX_THREADS = 128;

__device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z ^= z >> 30;
  z *= 0xBF58476D1CE4E5B9ull;
  z ^= z >> 27;
  z *= 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

__device__ __forceinline__ void add_word(uint64_t& h0, uint64_t& h1, uint64_t word, int64_t k, int tag) {
  const uint64_t p = (uint64_t)(4 * k + tag + 1) * PREFIX_GOLD;
  h0 += mix64(word ^ mix64(PREFIX_SEED0 + p));
  h1 += mix64(word ^ mix64(PREFIX_SEED1 + p));
}

// One CTA per row t.  Its cloud c is found by binary search of cu_rows, as knn_rows_paged_kernel finds it; its node is
// i = n_prev[c] + t - cu_rows[c], and its pair row starts at entry pair_off[c] + (t - cu_rows[c]) n_cur_c of the step's
// concatenated pair inputs.
__global__ void __launch_bounds__(PREFIX_THREADS) prefix_keys_kernel(
    const float* __restrict__ feats, int64_t width, const float* __restrict__ coors, const int64_t* __restrict__ edge_tokens,
    const float* __restrict__ edge_values, int edge_dim, const uint8_t* __restrict__ neighbor_mask,
    const int64_t* __restrict__ cu_rows, const int64_t* __restrict__ n_prev, const int64_t* __restrict__ pair_off, int num_clouds,
    uint64_t* __restrict__ out) {
  const int64_t t = blockIdx.x;
  int lo = 0, hi = num_clouds - 1;                  // the last cloud with cu_rows[lo] <= t
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (cu_rows[mid] <= t) lo = mid; else hi = mid - 1;
  }
  const int64_t r = t - cu_rows[lo];
  const int64_t i = n_prev[lo] + r;
  const int64_t n_cur = n_prev[lo] + cu_rows[lo + 1] - cu_rows[lo];
  const int64_t pair = (edge_tokens || edge_values || neighbor_mask) ? pair_off[lo] + r * n_cur : 0;
  uint64_t h0 = 0, h1 = 0;
  const float* f = feats + t * width;
  for (int64_t k = threadIdx.x; k < width; k += PREFIX_THREADS) add_word(h0, h1, __float_as_uint(f[k]), k, 0);
  if (threadIdx.x < 3) add_word(h0, h1, __float_as_uint(coors[3 * t + threadIdx.x]), threadIdx.x, 1);
  if (edge_tokens) {
    const int64_t* e = edge_tokens + pair;
    for (int64_t j = threadIdx.x; j < i; j += PREFIX_THREADS) add_word(h0, h1, (uint64_t)e[j], j, 2);
  } else if (edge_values) {
    const float* e = edge_values + pair * edge_dim;
    const int64_t n = i * edge_dim;
    for (int64_t k = threadIdx.x; k < n; k += PREFIX_THREADS) add_word(h0, h1, __float_as_uint(e[k]), k, 2);
  }
  if (neighbor_mask) {
    const uint8_t* m = neighbor_mask + pair;
    for (int64_t j = threadIdx.x; j < i; j += PREFIX_THREADS) add_word(h0, h1, m[j], j, 3);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    h0 += __shfl_xor_sync(0xffffffffu, h0, o);
    h1 += __shfl_xor_sync(0xffffffffu, h1, o);
  }
  __shared__ uint64_t part[2][PREFIX_THREADS / 32];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    part[0][warp] = h0;
    part[1][warp] = h1;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    uint64_t s0 = 0, s1 = 0;
#pragma unroll
    for (int w = 0; w < PREFIX_THREADS / 32; ++w) {
      s0 += part[0][w];
      s1 += part[1][w];
    }
    out[2 * t] = mix64(s0);
    out[2 * t + 1] = mix64(s1);
  }
}

}  // namespace
}  // namespace se3

extern "C" int se3_prefix_keys_fwd(const float* feats, int64_t rows, int64_t width, const float* coors, const int64_t* edge_tokens,
                                   const float* edge_values, int edge_dim, const uint8_t* neighbor_mask, const int64_t* cu_rows,
                                   const int64_t* n_prev, const int64_t* pair_off, int num_clouds, uint64_t* out, void* stream) {
  using namespace se3;
  SE3_REQUIRE(feats && coors && cu_rows && n_prev && out, "se3_prefix_keys_fwd: null pointer");
  SE3_REQUIRE(!(edge_tokens && edge_values), "se3_prefix_keys_fwd: give edge tokens or edge values, not both");
  SE3_REQUIRE(!(edge_tokens || edge_values || neighbor_mask) || pair_off, "se3_prefix_keys_fwd: pair inputs need pair_off");
  SE3_REQUIRE(!edge_values || edge_dim >= 1, "se3_prefix_keys_fwd: edge values need edge_dim >= 1 (got %d)", edge_dim);
  SE3_REQUIRE(num_clouds > 0 && rows >= num_clouds && rows < (1ll << 31),
              "se3_prefix_keys_fwd: need 0 < num_clouds <= rows < 2^31 (got %d clouds, %lld rows)", num_clouds, (long long)rows);
  SE3_REQUIRE(width >= 0, "se3_prefix_keys_fwd: width must be >= 0 (got %lld)", (long long)width);
  prefix_keys_kernel<<<(unsigned)rows, PREFIX_THREADS, 0, as_stream(stream)>>>(feats, width, coors, edge_tokens, edge_values, edge_dim,
                                                                               neighbor_mask, cu_rows, n_prev, pair_off, num_clouds, out);
  SE3_LAUNCH_OK();
  return SE3_OK;
}
