// K1: neighbour graph, pair-feature gather and masked-mean pooling.
//
// Replaces the dense [b,n,n-1] temporaries + torch.topk + batched_index_select of the reference
// (se3_transformer_pytorch.py:1171-1294, utils.py:56-80) with one CTA per query node that sorts (distance, column) keys of its
// row bitonically in shared memory and emits only the k winners.  A row of up to KNN_TILE columns is sorted whole; a longer one
// is walked in tiles of KNN_TILE columns, each merged into a running list of the best next_pow2(k) keys.  One kernel,
// knn_kernel, serves padded batches [b, n] and packed batches of clouds of different sizes, with pair masks given as bytes
// (DensePairs) or as sorted column lists (CsrPairs; pair_lookup_kernel finds a neighbour's pair in such a list).
#include "common.cuh"
#include <cfloat>
#include <algorithm>
#include <type_traits>
#include <vector>

namespace se3 {

constexpr int KNN_TILE = 4096;      // columns per shared-memory sort; also the largest k (the running list sits next to the tile)

__host__ __device__ inline int next_pow2(int v) {
  int p = 1;
  while (p < v) p <<= 1;
  return p;
}

__host__ __device__ inline int knn_npad(int n) {
  int npad = 2;
  while (npad < n - 1) npad <<= 1;
  return npad;
}

// Where the pair row of node i comes from.  DensePairs: row i of the cloud's [n, n] byte masks (or NULL).  CsrPairs: the sorted
// column lists of row i, staged tile by tile into shared-memory bitmaps.  Both answer, for a column j != i of the current tile,
// whether j is outside the neighbour mask and whether it is bonded; knn_tile_keys applies the answers in the same order.
struct DensePairs {
  const uint8_t* __restrict__ nbr;
  const uint8_t* __restrict__ adj;
  template <int THREADS>
  __device__ __forceinline__ void stage(int, int) {}
  __device__ __forceinline__ bool excluded(int j) const { return nbr && !nbr[j]; }
  __device__ __forceinline__ bool bonded(int j) const { return adj && adj[j]; }
};

constexpr int CSR_BITMAP_WORDS = KNN_TILE / 32 + 1;   // columns j in [t0, t0 + KNN_TILE] of one tile (self removed: one extra)

// first position p in [lo, hi) with cols[p] >= v (hi if none)
__device__ __forceinline__ int64_t csr_lower_bound(const int* __restrict__ cols, int64_t lo, int64_t hi, int v) {
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (cols[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

struct CsrPairs {
  const int* __restrict__ nbr;       // columns of the neighbour mask (NULL: no mask); row entries [nbr_lo, nbr_hi)
  const int* __restrict__ adj;       // columns of the bonded neighbours (NULL: none); row entries [adj_lo, adj_hi)
  int64_t nbr_lo, nbr_hi, adj_lo, adj_hi;
  unsigned* bits;                    // 2 x CSR_BITMAP_WORDS words of shared memory: neighbour mask, then bonded
  int t0;

  template <int THREADS>
  __device__ __forceinline__ void scatter(const int* __restrict__ cols, int64_t lo, int64_t hi, unsigned* words, int width) {
    // only the row's entries inside this tile are read; an entry outside [t0, t0 + width] never touches the bitmap
    const int64_t first = csr_lower_bound(cols, lo, hi, t0);
    for (int64_t p = first + threadIdx.x; p < hi; p += THREADS) {
      const int c = cols[p];
      if (c > t0 + width) break;
      if (c >= t0) atomicOr(&words[(c - t0) >> 5], 1u << ((c - t0) & 31));
    }
  }
  // bits <- the row's entries among the columns of tile [t0, t0 + width) (self-removed positions, so columns t0 .. t0 + width)
  template <int THREADS>
  __device__ __forceinline__ void stage(int tile0, int width) {
    t0 = tile0;
    for (int w = threadIdx.x; w < 2 * CSR_BITMAP_WORDS; w += THREADS) bits[w] = 0u;
    __syncthreads();
    if (nbr) scatter<THREADS>(nbr, nbr_lo, nbr_hi, bits, width);
    if (adj) scatter<THREADS>(adj, adj_lo, adj_hi, bits + CSR_BITMAP_WORDS, width);
    __syncthreads();
  }
  __device__ __forceinline__ bool bit(const unsigned* words, int j) const { return (words[(j - t0) >> 5] >> ((j - t0) & 31)) & 1u; }
  __device__ __forceinline__ bool excluded(int j) const { return nbr && !bit(bits, j); }
  __device__ __forceinline__ bool bonded(int j) const { return adj && bit(bits + CSR_BITMAP_WORDS, j); }
};

// Where column j of a cloud keeps its coordinates.  Flat (const float* c): row j of the cloud's [n, 3] block, neighbour index
// j_base + j.  PagedCoords: row pages[toff + j / P] P + j % P of a pool of pages of P nodes ([pages, P, 3]; pages[toff ..]: the
// cloud's page ids in order); its neighbour index is the column j, which knn_rows_paged_kernel turns into the pool row.  Only the
// address of a column differs: keys, ties and distances are the same, so a paged row is bit for bit the flat row of the same
// cloud.  j / P is a multiply-high and a shift (page_divisor): with it, and with no pointer to the column output carried
// through the search, the paged search fits 40 registers without spilling.
struct PagedCoords {
  const float* __restrict__ pool;
  const int* __restrict__ pages;
  int toff;
  unsigned P, magic, shift;
  __device__ __forceinline__ int64_t row(int j) const {
    const unsigned q = (__umulhi((unsigned)j, magic) + (unsigned)j) >> shift;       // j / P for 0 <= j < 2^31
    return (int64_t)pages[toff + q] * P + ((unsigned)j - q * P);
  }
};

// magic, shift with (umulhi(j, magic) + j) >> shift = j / P for 0 <= j < 2^31 (Granlund and Montgomery, 1994): shift =
// ceil(log2 P), magic = floor(2^32 (2^shift - P) / P) + 1.  The sum stays below 2^32 because umulhi(j, magic) < j < 2^31.
static inline void page_divisor(unsigned P, unsigned& magic, unsigned& shift) {
  shift = 0;
  while ((1ull << shift) < P) ++shift;
  magic = (unsigned)((((1ull << shift) - P) << 32) / P + 1);
}
__device__ __forceinline__ float coord(const float* __restrict__ c, int j, int d) { return c[j * 3 + d]; }
__device__ __forceinline__ float coord(const PagedCoords& c, int j, int d) { return c.pool[c.row(j) * 3 + d]; }
__device__ __forceinline__ void emit(const float* __restrict__, int64_t* __restrict__ out_idx, int r, int64_t j_base, int j) {
  out_idx[r] = j_base + j;
}
__device__ __forceinline__ void emit(const PagedCoords&, int64_t* __restrict__ out_idx, int r, int64_t, int j) { out_idx[r] = j; }

// keys[0, width) <- the keys of the self-removed columns [t0, t0 + width) of row i, ~0 past the last column.
// key = (bits(modified distance) << 32) | column.  Distances are >= 0 so the IEEE bit pattern is order preserving; equal
// distances order by column, which is the stable-argsort tie rule the oracle uses (torch.topk leaves ties unspecified).
// Returns whether this thread wrote a key below `kth`.
template <int THREADS, class Pairs, class Coords>
__device__ __forceinline__ bool knn_tile_keys(unsigned long long* keys, const Coords c, int n, int i, float xi,
                                              float yi, float zi, int t0, int width, const Pairs& pairs, int causal,
                                              unsigned long long kth) {
  bool below = false;
  for (int t = threadIdx.x; t < width; t += THREADS) {
    const int jc = t0 + t;
    unsigned long long key = ~0ull;
    if (jc < n - 1) {
      const int j = jc + (jc >= i);
      const float dx = xi - coord(c, j, 0), dy = yi - coord(c, j, 1), dz = zi - coord(c, j, 2);
      float d = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
      if (pairs.excluded(j)) d = FLT_MAX;
      if (pairs.bonded(j)) d = 0.f;
      if (causal && jc >= i) d = FLT_MAX;
      key = ((unsigned long long)__float_as_uint(d) << 32) | (unsigned)jc;
    }
    keys[t] = key;
    below |= key < kth;
  }
  return below;
}

// bitonic sort of keys[0, npad), ascending; npad a power of two
template <int THREADS>
__device__ __forceinline__ void knn_sort(unsigned long long* keys, int npad) {
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
}

// The neighbour list of node i of one cloud of n nodes (c = where its coordinates are, see coord); the same body for every cloud
// form and pair form of knn_kernel, so that all produce the same bits.  pairs:
// row i of the cloud's pair masks (DensePairs or CsrPairs); node_mask: the cloud's [n] node mask (or NULL).  Writes slots
// [0, K_out) of the row at out_*; slots r >= k are copies of slot k - 1 with mask 0, and indices are those of emit.
// keys: npad = next_pow2(n - 1) keys of shared memory when n - 1 <= KNN_TILE (one sort of the whole row), otherwise
// KNN_TILE + next_pow2(k) keys (tile, then running list).  Keys are unique, so every top-k order gives the bits of one full sort.
template <int THREADS, class Pairs, class Coords>
__device__ __forceinline__ void knn_row(unsigned long long* keys, const Coords c, int n, int i, int k, int npad,
                                        Pairs pairs, const uint8_t* __restrict__ node_mask, float valid_radius, int causal, int K_out,
                                        int64_t j_base, int64_t* __restrict__ out_idx, uint8_t* __restrict__ out_mask,
                                        float* __restrict__ out_rel_pos, float* __restrict__ out_rel_dist) {
  const float xi = coord(c, i, 0), yi = coord(c, i, 1), zi = coord(c, i, 2);
  const unsigned long long* best = keys;
  if (n - 1 <= KNN_TILE) {
    pairs.template stage<THREADS>(0, npad);
    knn_tile_keys<THREADS>(keys, c, n, i, xi, yi, zi, 0, npad, pairs, causal, 0ull);
    __syncthreads();
    knn_sort<THREADS>(keys, npad);
  } else {
    unsigned long long* list = keys + KNN_TILE;      // the kpad smallest keys of the tiles so far, ascending
    const int kpad = next_pow2(k);
    for (int t = threadIdx.x; t < kpad; t += THREADS) list[t] = ~0ull;
    for (int t0 = 0; t0 < n - 1; t0 += KNN_TILE) {
      const unsigned long long kth = t0 ? list[k - 1] : ~0ull;
      pairs.template stage<THREADS>(t0, KNN_TILE);
      const bool below = knn_tile_keys<THREADS>(keys, c, n, i, xi, yi, zi, t0, KNN_TILE, pairs, causal, kth);
      if (__syncthreads_count(below) == 0) continue;   // nothing in this tile beats the current k-th key
      knn_sort<THREADS>(keys, KNN_TILE);
      // bitonic merge: min of the ascending list and the tile's first kpad keys reversed is a bitonic sequence of the kpad
      // smallest keys of both; log2(kpad) half-cleaner stages sort it
      for (int t = threadIdx.x; t < kpad; t += THREADS) list[t] = min(list[t], keys[kpad - 1 - t]);
      __syncthreads();
      for (int stride = kpad >> 1; stride > 0; stride >>= 1) {
        for (int t = threadIdx.x; t < (kpad >> 1); t += THREADS) {
          const int lo = 2 * t - (t & (stride - 1));
          const int hi = lo + stride;
          const unsigned long long a = list[lo], bb = list[hi];
          if (a > bb) { list[lo] = bb; list[hi] = a; }
        }
        __syncthreads();
      }
    }
    best = list;
  }
  const bool mi = node_mask ? node_mask[i] != 0 : true;
  for (int r = threadIdx.x; r < K_out; r += THREADS) {
    const unsigned long long key = best[r < k ? r : k - 1];
    const int jc = (int)(key & 0xffffffffu);
    const float dmod = __uint_as_float((unsigned)(key >> 32));
    const int j = jc + (jc >= i);
    const float dx = xi - coord(c, j, 0), dy = yi - coord(c, j, 1), dz = zi - coord(c, j, 2);
    const float d = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
    bool m = r < k && dmod <= valid_radius;
    if (node_mask) m = m && mi && node_mask[j] != 0;
    emit(c, out_idx, r, j_base, j);
    out_mask[r] = m ? 1 : 0;
    out_rel_pos[r * 3 + 0] = dx;
    out_rel_pos[r * 3 + 1] = dy;
    out_rel_pos[r * 3 + 2] = dz;
    out_rel_dist[r] = d;
  }
}

// Row pointers of row r of a column list, clamped to [0, nnz] so that a malformed list reads no memory outside it.
__device__ __forceinline__ void csr_bounds(const se3_pairs& p, int64_t r, int64_t& lo, int64_t& hi) {
  lo = min(max(p.row_ptr[r], (int64_t)0), p.nnz);
  hi = min(max(p.row_ptr[r + 1], lo), p.nnz);
}

// One CTA per node t of the flat node list.  Uniform clouds (cu_seqlens NULL): cloud c = t / n of n nodes, K = k, indices
// local to the cloud.  Packed clouds: the CTA finds its cloud by binary search in cu_seqlens, searches it for k_per_cloud[c]
// neighbours and writes K >= k_c slots with global indices; dense pair masks are the clouds' [n_c, n_c] matrices flattened
// end to end, cloud c starting at pair_off[c].  A shared pair input (one matrix or list for every cloud) is read at row i.
// Shared memory: key_words keys (see knn_row), then the two bitmaps of CsrPairs.  Both instantiations ask for 6 CTAs per SM:
// without it the tiled branch of knn_row raises them from 40 to 48 registers, and whole-row searches would lose a CTA per SM.
template <int THREADS, class Pairs>
__global__ void __launch_bounds__(THREADS, 6)
knn_kernel(const float* __restrict__ coors, const int64_t* __restrict__ cu_seqlens, const int* __restrict__ k_per_cloud,
           const int64_t* __restrict__ pair_off, const uint8_t* __restrict__ node_mask, const se3_pairs nbr, const se3_pairs adj,
           int num_clouds, int n, int K, int key_words, float valid_radius, int causal,
           int64_t* __restrict__ out_idx, uint8_t* __restrict__ out_mask,
           float* __restrict__ out_rel_pos, float* __restrict__ out_rel_dist) {
  extern __shared__ unsigned long long keys[];
  const int64_t t = blockIdx.x;
  int64_t start, base;                              // first node of the cloud, start of its dense pair matrix
  int n_c, k_c;
  if (cu_seqlens) {
    int lo = 0, hi = num_clouds - 1;                // the last cloud c with cu_seqlens[c] <= t
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (cu_seqlens[mid] <= t) lo = mid; else hi = mid - 1;
    }
    start = cu_seqlens[lo];
    n_c = (int)(cu_seqlens[lo + 1] - start);
    k_c = k_per_cloud[lo];
    base = pair_off ? pair_off[lo] : 0;
  } else {
    start = t / n * n;
    n_c = n;
    k_c = K;
    base = start * n;
  }
  const int i = (int)(t - start);
  Pairs pairs;
  if constexpr (std::is_same<Pairs, DensePairs>::value) {
    const int64_t row = (int64_t)i * n_c;
    pairs = DensePairs{nbr.dense ? nbr.dense + (nbr.shared ? 0 : base) + row : nullptr,
                       adj.dense ? adj.dense + (adj.shared ? 0 : base) + row : nullptr};
  } else {
    pairs = CsrPairs{nbr.cols, adj.cols, 0, 0, 0, 0, reinterpret_cast<unsigned*>(keys + key_words), 0};
    if (nbr.cols) csr_bounds(nbr, nbr.shared ? i : t, pairs.nbr_lo, pairs.nbr_hi);
    if (adj.cols) csr_bounds(adj, adj.shared ? i : t, pairs.adj_lo, pairs.adj_hi);
  }
  const int64_t o = t * K;
  knn_row<THREADS>(keys, coors + start * 3, n_c, i, k_c, knn_npad(n_c), pairs, node_mask ? node_mask + start : nullptr,
                   valid_radius, causal, K, cu_seqlens ? start : 0, out_idx + o, out_mask + o, out_rel_pos + o * 3,
                   out_rel_dist + o);
}

// One CTA per new row of clouds that grow one step at a time, stored with a leading dimension of ld nodes (coors [rows, ld, 3],
// node_mask [rows, ld]).  Uniform clouds (cu_rows NULL): rows [row0, row0 + nrows) of b clouds whose first n nodes are searched
// for k neighbours, nbr [b, nrows, n] the new rows' byte masks, indices local to the cloud.  Ragged clouds: the CTA finds its
// cloud c by binary search in cu_rows, as knn_kernel does in cu_seqlens; its row r is node n_prev[c] + r of the cloud in store
// row slot[c], searched over its first n_prev[c] + m_c nodes for k_per_cloud[c] neighbours into k >= k_c slots; its byte mask
// row starts at nbr + pair_off[c] + r (n_prev[c] + m_c) (pair_off[c] < 0: no mask); indices are slot[c] ld + j.  The row body
// is knn_row, so the results are those of knn_kernel's rows.
template <int THREADS>
__global__ void __launch_bounds__(THREADS, 6)
knn_rows_kernel(const float* __restrict__ coors, const uint8_t* __restrict__ node_mask, const uint8_t* __restrict__ nbr,
                const int64_t* __restrict__ cu_rows, const int64_t* __restrict__ slot, const int64_t* __restrict__ n_prev,
                const int64_t* __restrict__ k_per_cloud, const int64_t* __restrict__ pair_off, int num_clouds, int n, int64_t ld,
                int row0, int nrows, int k, float valid_radius, int causal, int64_t* __restrict__ out_idx,
                uint8_t* __restrict__ out_mask, float* __restrict__ out_rel_pos, float* __restrict__ out_rel_dist) {
  extern __shared__ unsigned long long keys[];
  const int64_t t = blockIdx.x;
  int64_t c, j_base = 0;
  int i, n_c, k_c;
  const uint8_t* row_mask;
  if (cu_rows) {
    int lo = 0, hi = num_clouds - 1;                // the last cloud with cu_rows[lo] <= t
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (cu_rows[mid] <= t) lo = mid; else hi = mid - 1;
    }
    const int64_t r = t - cu_rows[lo];
    c = slot[lo];
    i = (int)(n_prev[lo] + r);
    n_c = (int)(n_prev[lo] + cu_rows[lo + 1] - cu_rows[lo]);
    k_c = (int)k_per_cloud[lo];
    row_mask = nbr && pair_off[lo] >= 0 ? nbr + pair_off[lo] + r * n_c : nullptr;
    j_base = c * ld;
  } else {
    c = t / nrows;
    i = row0 + (int)(t % nrows);
    n_c = n;
    k_c = k;
    row_mask = nbr ? nbr + t * n : nullptr;
  }
  const int64_t o = t * k;
  knn_row<THREADS>(keys, coors + c * ld * 3, n_c, i, k_c, knn_npad(n_c), DensePairs{row_mask, nullptr},
                   node_mask ? node_mask + c * ld : nullptr, valid_radius, causal, k, j_base, out_idx + o, out_mask + o,
                   out_rel_pos + o * 3, out_rel_dist + o);
}

// The ragged form of knn_rows_kernel for clouds kept in pages of P nodes of one pool, coors [pages, P, 3] (PagedCausalDecoder):
// cloud c's page ids are pages[table_off[c] ..], and its node j is pool row pages[table_off[c] + j / P] P + j % P.  out_idx
// gets that pool row, out_col the column j; everything else is as in knn_rows_kernel.  table_off < 2^31.
// BUCKET (a decoding step replayed from a CUDA graph): the grid has a fixed number of CTAs, at least the step's rows M =
// cu_rows[num_clouds], and clouds past the step's are empty (cu_rows = M).  CTA t >= M is a padding row: it repeats the search
// of row M - 1 and writes its own output row t.
template <int THREADS, bool BUCKET>
__global__ void __launch_bounds__(THREADS, 6)
knn_rows_paged_kernel(const float* __restrict__ pool, const int* __restrict__ pages, const uint8_t* __restrict__ nbr,
                      const int64_t* __restrict__ cu_rows, const int64_t* __restrict__ n_prev, const int64_t* __restrict__ k_per_cloud,
                      const int64_t* __restrict__ pair_off, const int64_t* __restrict__ table_off, int num_clouds, unsigned P,
                      unsigned magic, unsigned shift, int K, float valid_radius, int causal, int64_t* __restrict__ out_idx, int64_t* __restrict__ out_col,
                      uint8_t* __restrict__ out_mask, float* __restrict__ out_rel_pos, float* __restrict__ out_rel_dist) {
  extern __shared__ unsigned long long keys[];
  int64_t t = blockIdx.x;
  if constexpr (BUCKET) t = min(t, cu_rows[num_clouds] - 1);
  int lo = 0, hi = num_clouds - 1;                  // the last cloud with cu_rows[lo] <= t
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (cu_rows[mid] <= t) lo = mid; else hi = mid - 1;
  }
  const int64_t r = t - cu_rows[lo];
  const int i = (int)(n_prev[lo] + r);
  const int n_c = (int)(n_prev[lo] + cu_rows[lo + 1] - cu_rows[lo]);
  const uint8_t* row_mask = nbr && pair_off[lo] >= 0 ? nbr + pair_off[lo] + r * n_c : nullptr;
  const int64_t o = (BUCKET ? (int64_t)blockIdx.x : t) * K;
  const PagedCoords c{pool, pages, (int)table_off[lo], P, magic, shift};
  knn_row<THREADS>(keys, c, n_c, i, (int)k_per_cloud[lo], knn_npad(n_c), DensePairs{row_mask, nullptr}, nullptr, valid_radius,
                   causal, K, 0, out_idx + o, out_mask + o, out_rel_pos + o * 3, out_rel_dist + o);
  for (int s = threadIdx.x; s < K; s += THREADS) {  // the slots this thread wrote in knn_row: columns -> pool rows
    const int j = (int)out_idx[o + s];
    out_col[o + s] = j;
    out_idx[o + s] = c.row(j);
  }
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

// out[s] = position of column idx[s] in CSR row s / k (clamped to [0, nnz] as in csr_bounds), or -1 if the row lacks it.
__global__ void pair_lookup_kernel(const int64_t* __restrict__ ptr, const int* __restrict__ cols, int64_t nnz, int64_t stride,
                                   const int64_t* __restrict__ idx, int n, int k, int64_t total, int64_t* __restrict__ out) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= total) return;
  const int64_t bi = s / k;                  // b * n + i
  const int64_t r = (bi / n) * stride + bi % n;
  const int64_t lo = min(max(ptr[r], (int64_t)0), nnz), hi = min(max(ptr[r + 1], lo), nnz);
  const int64_t j = idx[s];
  int64_t pos = -1;
  if (j >= 0 && j < n) {
    const int64_t p = csr_lower_bound(cols, lo, hi, (int)j);
    if (p < hi && cols[p] == (int)j) pos = p;
  }
  out[s] = pos;
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

extern "C" int se3_knn_fwd(const float* coors, const int64_t* cu_seqlens, const int* k_per_cloud, const int64_t* pair_off,
                           const uint8_t* node_mask, const se3_pairs* neighbor_mask, const se3_pairs* sparse_adj, int b, int64_t n,
                           int k, float valid_radius, int causal, int64_t* out_idx, uint8_t* out_mask, float* out_rel_pos,
                           float* out_rel_dist, void* stream) {
  using namespace se3;
  const se3_pairs none{nullptr, nullptr, nullptr, 0, 0};
  const se3_pairs& nbr = neighbor_mask ? *neighbor_mask : none;
  const se3_pairs& adj = sparse_adj ? *sparse_adj : none;
  const bool dense = nbr.dense || adj.dense, csr = nbr.cols || adj.cols;
  SE3_REQUIRE(!(dense && csr), "se3_knn_fwd: the pair masks must both be dense or both be column lists");
  for (const se3_pairs* p : {&nbr, &adj})
    SE3_REQUIRE(!p->cols || (p->row_ptr && p->nnz >= 0), "se3_knn_fwd: a column list needs row pointers and nnz >= 0");
  const int64_t nodes = cu_seqlens ? n : (int64_t)b * n;
  SE3_REQUIRE(nodes < (1ll << 31), "se3_knn_fwd: %lld nodes exceed the 1-D grid", (long long)nodes);
  cudaStream_t s = as_stream(stream);
  int n_max = (int)n;                               // nodes of the largest cloud
  if (!cu_seqlens) {
    SE3_REQUIRE(b > 0 && n > 1, "se3_knn_fwd: need b > 0 and n > 1 (got b=%d n=%lld)", b, (long long)n);
    SE3_REQUIRE(k >= 1 && k <= n - 1, "se3_knn_fwd: k must be in [1, n-1] (got k=%d n=%lld)", k, (long long)n);
    SE3_REQUIRE(k <= KNN_TILE, "se3_knn_fwd: k = %d neighbours exceeds %d, the longest list the tiled search keeps in shared memory",
                k, KNN_TILE);
  } else {
    SE3_REQUIRE(!csr && !node_mask && !nbr.shared && !adj.shared,
                "se3_knn_fwd: packed clouds take neither column lists, a node mask nor a shared pair mask");
    SE3_REQUIRE(b > 0 && n > 0 && k > 0, "se3_knn_fwd: need num_clouds, total, K > 0 (got %d, %lld, %d)", b, (long long)n, k);
    SE3_REQUIRE(!dense || pair_off, "se3_knn_fwd: dense pair masks of packed clouds need pair_off");
    // the sizes live on the device: read them back once (a few hundred bytes) so that a bad batch is refused, not read out of bounds
    std::vector<int64_t> cu(b + 1), off(b);
    std::vector<int> kc(b);
    SE3_CUDA_OK(cudaMemcpyAsync(cu.data(), cu_seqlens, cu.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    SE3_CUDA_OK(cudaMemcpyAsync(kc.data(), k_per_cloud, kc.size() * sizeof(int), cudaMemcpyDeviceToHost, s));
    if (dense) SE3_CUDA_OK(cudaMemcpyAsync(off.data(), pair_off, off.size() * sizeof(int64_t), cudaMemcpyDeviceToHost, s));
    SE3_CUDA_OK(cudaStreamSynchronize(s));
    SE3_REQUIRE(cu[0] == 0 && cu[b] == n, "se3_knn_fwd: cu_seqlens must run from 0 to total = %lld (got %lld .. %lld)",
                (long long)n, (long long)cu[0], (long long)cu[b]);
    int64_t pairs_before = 0;
    n_max = 0;
    for (int c = 0; c < b; ++c) {
      const int64_t n_c = cu[c + 1] - cu[c];
      SE3_REQUIRE(n_c >= 2 && n_c - 1 <= KNN_TILE, "se3_knn_fwd: cloud %d has %lld nodes; each cloud needs 2 .. 4097", c, (long long)n_c);
      SE3_REQUIRE(kc[c] >= 1 && kc[c] <= n_c - 1, "se3_knn_fwd: k of cloud %d must be in [1, n_c - 1] (got k=%d n_c=%lld)", c,
                  kc[c], (long long)n_c);
      SE3_REQUIRE(kc[c] <= k, "se3_knn_fwd: K = %d is smaller than k = %d of cloud %d", k, kc[c], c);
      SE3_REQUIRE(!dense || off[c] == pairs_before, "se3_knn_fwd: pair_off[%d] = %lld, expected sum of n_c^2 before it = %lld", c,
                  (long long)off[c], (long long)pairs_before);
      pairs_before += n_c * n_c;
      n_max = std::max(n_max, (int)n_c);
    }
  }
  constexpr int THREADS = 256;
  const int key_words = n_max - 1 > KNN_TILE ? KNN_TILE + next_pow2(k) : knn_npad(n_max);
  const size_t smem = (size_t)key_words * sizeof(unsigned long long) + (csr ? 2 * CSR_BITMAP_WORDS * sizeof(unsigned) : 0);
  auto launch = [&](auto kernel) -> int {
    if (smem > 48 * 1024) SE3_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<(unsigned)nodes, THREADS, smem, s>>>(coors, cu_seqlens, k_per_cloud, pair_off, node_mask, nbr, adj, b, (int)n, k,
                                                  key_words, valid_radius, causal, out_idx, out_mask, out_rel_pos, out_rel_dist);
    SE3_LAUNCH_OK();
    return SE3_OK;
  };
  return csr ? launch(knn_kernel<THREADS, CsrPairs>) : launch(knn_kernel<THREADS, DensePairs>);
}

namespace se3 {
// knn_rows_kernel over `rows` CTAs; n: the longest searched cloud, which sizes shared memory (K slots per row)
static int launch_knn_rows(const float* coors, const uint8_t* node_mask, const uint8_t* nbr, const int64_t* cu_rows,
                           const int64_t* slot, const int64_t* n_prev, const int64_t* k_per_cloud, const int64_t* pair_off,
                           int num_clouds, int n, int64_t ld, int row0, int nrows, int64_t rows, int K, float valid_radius, int causal,
                           int64_t* out_idx, uint8_t* out_mask, float* out_rel_pos, float* out_rel_dist, void* stream) {
  constexpr int THREADS = 256;
  const int key_words = n - 1 > KNN_TILE ? KNN_TILE + next_pow2(K) : knn_npad(n);
  const size_t smem = (size_t)key_words * sizeof(unsigned long long);
  auto kernel = knn_rows_kernel<THREADS>;
  if (smem > 48 * 1024) SE3_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<(unsigned)rows, THREADS, smem, as_stream(stream)>>>(coors, node_mask, nbr, cu_rows, slot, n_prev, k_per_cloud, pair_off,
                                                               num_clouds, n, ld, row0, nrows, K, valid_radius, causal, out_idx,
                                                               out_mask, out_rel_pos, out_rel_dist);
  SE3_LAUNCH_OK();
  return SE3_OK;
}
}  // namespace se3

extern "C" int se3_knn_rows_fwd(const float* coors, const uint8_t* node_mask, const uint8_t* neighbor_mask, int b, int64_t n, int64_t ld,
                                int row0, int nrows, int k, float valid_radius, int causal, int64_t* out_idx, uint8_t* out_mask,
                                float* out_rel_pos, float* out_rel_dist, void* stream) {
  using namespace se3;
  SE3_REQUIRE(coors && out_idx && out_mask && out_rel_pos && out_rel_dist, "se3_knn_rows_fwd: null pointer");
  SE3_REQUIRE(b > 0 && n > 1 && n < (1ll << 31) && ld >= n, "se3_knn_rows_fwd: need b > 0, 1 < n < 2^31, ld >= n (got b=%d n=%lld ld=%lld)",
              b, (long long)n, (long long)ld);
  SE3_REQUIRE(row0 >= 0 && nrows >= 1 && row0 + (int64_t)nrows <= n, "se3_knn_rows_fwd: rows [%d, %d + %d) outside the %lld nodes", row0,
              row0, nrows, (long long)n);
  SE3_REQUIRE(k >= 1 && k <= n - 1 && k <= KNN_TILE, "se3_knn_rows_fwd: k must be in [1, min(n-1, %d)] (got k=%d n=%lld)", KNN_TILE, k,
              (long long)n);
  SE3_REQUIRE((int64_t)b * nrows < (1ll << 31), "se3_knn_rows_fwd: %lld rows exceed the 1-D grid", (long long)b * nrows);
  return launch_knn_rows(coors, node_mask, neighbor_mask, nullptr, nullptr, nullptr, nullptr, nullptr, 0, (int)n, ld, row0, nrows,
                         (int64_t)b * nrows, k, valid_radius, causal, out_idx, out_mask, out_rel_pos, out_rel_dist, stream);
}

extern "C" int se3_knn_rows_packed_fwd(const float* coors, const uint8_t* neighbor_mask, const int64_t* cu_rows, const int64_t* slot,
                                       const int64_t* n_prev, const int64_t* k_per_cloud, const int64_t* pair_off, int num_clouds,
                                       int64_t rows, int64_t ld, int n_max, int K, float valid_radius, int causal, int64_t* out_idx,
                                       uint8_t* out_mask, float* out_rel_pos, float* out_rel_dist, void* stream) {
  using namespace se3;
  SE3_REQUIRE(coors && cu_rows && slot && n_prev && k_per_cloud && out_idx && out_mask && out_rel_pos && out_rel_dist,
              "se3_knn_rows_packed_fwd: null pointer");
  SE3_REQUIRE(!neighbor_mask || pair_off, "se3_knn_rows_packed_fwd: a neighbour mask needs pair_off");
  SE3_REQUIRE(num_clouds > 0 && rows >= num_clouds && rows < (1ll << 31),
              "se3_knn_rows_packed_fwd: need 0 < num_clouds <= rows < 2^31 (got %d clouds, %lld rows)", num_clouds, (long long)rows);
  SE3_REQUIRE(n_max > 1 && n_max <= ld, "se3_knn_rows_packed_fwd: need 1 < n_max <= ld (got n_max=%d ld=%lld)", n_max, (long long)ld);
  SE3_REQUIRE(K >= 1 && K <= KNN_TILE, "se3_knn_rows_packed_fwd: K must be in [1, %d] (got %d)", KNN_TILE, K);
  return launch_knn_rows(coors, nullptr, neighbor_mask, cu_rows, slot, n_prev, k_per_cloud, pair_off, num_clouds, n_max, ld, 0, 1,
                         rows, K, valid_radius, causal, out_idx, out_mask, out_rel_pos, out_rel_dist, stream);
}

namespace se3 {
// knn_rows_paged_kernel over `rows` CTAs; n_max: the longest searched cloud, which sizes shared memory (K slots per row)
template <bool BUCKET>
static int launch_knn_rows_paged(const float* pool, const int* pages, const uint8_t* nbr, const int64_t* cu_rows,
                                 const int64_t* n_prev, const int64_t* k_per_cloud, const int64_t* pair_off, const int64_t* table_off,
                                 int num_clouds, int64_t rows, int page_size, int n_max, int K, float valid_radius, int causal,
                                 int64_t* out_idx, int64_t* out_col, uint8_t* out_mask, float* out_rel_pos, float* out_rel_dist,
                                 void* stream) {
  constexpr int THREADS = 256;
  const int key_words = n_max - 1 > KNN_TILE ? KNN_TILE + next_pow2(K) : knn_npad(n_max);
  const size_t smem = (size_t)key_words * sizeof(unsigned long long);
  unsigned magic, shift;
  page_divisor((unsigned)page_size, magic, shift);
  auto kernel = knn_rows_paged_kernel<THREADS, BUCKET>;
  if (smem > 48 * 1024) SE3_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<(unsigned)rows, THREADS, smem, as_stream(stream)>>>(pool, pages, nbr, cu_rows, n_prev, k_per_cloud, pair_off, table_off,
                                                               num_clouds, (unsigned)page_size, magic, shift, K, valid_radius, causal,
                                                               out_idx, out_col, out_mask, out_rel_pos, out_rel_dist);
  SE3_LAUNCH_OK();
  return SE3_OK;
}

// One thread per row t of a decoding step padded to `rows` rows (see se3_decode_plan_fwd).  The row's cloud is found as
// knn_rows_paged_kernel finds it, and its pool row with the same PagedCoords::row, so the plan and the search agree on every
// row; padding rows t >= M take row M - 1's position, cloud and pair row, and scratch pool row scratch_row + t - M.
__global__ void decode_plan_kernel(const int64_t* __restrict__ desc, int num_clouds, int rows, unsigned P, unsigned magic,
                                   unsigned shift, int64_t scratch_row, int64_t* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= rows) return;
  const int64_t* cu_rows = desc;
  const int64_t* n_prev = desc + num_clouds + 1;
  const int64_t* pair_off = desc + 3 * num_clouds + 1;
  const int64_t* table_off = desc + 4 * num_clouds + 1;
  const int* pages = reinterpret_cast<const int*>(desc + 5 * num_clouds + 1);
  const int64_t M = cu_rows[num_clouds];
  const int64_t s = min((int64_t)t, M - 1);
  int lo = 0, hi = num_clouds - 1;                  // the last cloud with cu_rows[lo] <= s
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (cu_rows[mid] <= s) lo = mid; else hi = mid - 1;
  }
  const int64_t r = s - cu_rows[lo];
  const int64_t n_cur = n_prev[lo] + cu_rows[lo + 1] - cu_rows[lo];
  const int pos = (int)(n_prev[lo] + r);
  const PagedCoords c{nullptr, pages, (int)table_off[lo], P, magic, shift};
  out[t] = pos;
  out[rows + t] = t < M ? c.row(pos) : scratch_row + (t - M);
  out[2 * rows + t] = pair_off[lo] + r * n_cur;
  out[3 * rows + t] = lo;
}
}  // namespace se3

extern "C" int se3_knn_rows_paged_fwd(const float* pool, const int* pages, const uint8_t* neighbor_mask, const int64_t* cu_rows,
                                      const int64_t* n_prev, const int64_t* k_per_cloud, const int64_t* pair_off,
                                      const int64_t* table_off, int num_clouds, int64_t rows, int page_size, int n_max, int K,
                                      float valid_radius, int causal, int64_t* out_idx, int64_t* out_col, uint8_t* out_mask,
                                      float* out_rel_pos, float* out_rel_dist, void* stream) {
  using namespace se3;
  SE3_REQUIRE(pool && pages && cu_rows && n_prev && k_per_cloud && table_off && out_idx && out_col && out_mask && out_rel_pos &&
              out_rel_dist, "se3_knn_rows_paged_fwd: null pointer");
  SE3_REQUIRE(!neighbor_mask || pair_off, "se3_knn_rows_paged_fwd: a neighbour mask needs pair_off");
  SE3_REQUIRE(num_clouds > 0 && rows >= num_clouds && rows < (1ll << 31),
              "se3_knn_rows_paged_fwd: need 0 < num_clouds <= rows < 2^31 (got %d clouds, %lld rows)", num_clouds, (long long)rows);
  SE3_REQUIRE(page_size >= 1, "se3_knn_rows_paged_fwd: page_size must be >= 1 (got %d)", page_size);
  SE3_REQUIRE(n_max > 1, "se3_knn_rows_paged_fwd: need n_max > 1 (got %d)", n_max);
  SE3_REQUIRE(K >= 1 && K <= KNN_TILE, "se3_knn_rows_paged_fwd: K must be in [1, %d] (got %d)", KNN_TILE, K);
  return launch_knn_rows_paged<false>(pool, pages, neighbor_mask, cu_rows, n_prev, k_per_cloud, pair_off, table_off, num_clouds, rows,
                                      page_size, n_max, K, valid_radius, causal, out_idx, out_col, out_mask, out_rel_pos,
                                      out_rel_dist, stream);
}

extern "C" int se3_decode_plan_fwd(const int64_t* desc, int num_clouds, int rows, int page_size, int64_t scratch_row, int64_t* out,
                                   void* stream) {
  using namespace se3;
  SE3_REQUIRE(desc && out, "se3_decode_plan_fwd: null pointer");
  SE3_REQUIRE(num_clouds > 0 && rows >= num_clouds, "se3_decode_plan_fwd: need 0 < num_clouds <= rows (got %d clouds, %d rows)",
              num_clouds, rows);
  SE3_REQUIRE(page_size >= 1 && scratch_row >= 0, "se3_decode_plan_fwd: need page_size >= 1 and scratch_row >= 0 (got %d, %lld)",
              page_size, (long long)scratch_row);
  unsigned magic, shift;
  page_divisor((unsigned)page_size, magic, shift);
  const int threads = 128;
  decode_plan_kernel<<<(unsigned)ceil_div(rows, threads), threads, 0, as_stream(stream)>>>(desc, num_clouds, rows, (unsigned)page_size,
                                                                                           magic, shift, scratch_row, out);
  SE3_LAUNCH_OK();
  return SE3_OK;
}

extern "C" int se3_knn_rows_paged_bucket_fwd(const float* pool, const int64_t* desc, const uint8_t* neighbor_mask, int num_clouds,
                                             int rows, int page_size, int n_max, int K, float valid_radius, int causal,
                                             int64_t* out_idx, int64_t* out_col, uint8_t* out_mask, float* out_rel_pos,
                                             float* out_rel_dist, void* stream) {
  using namespace se3;
  SE3_REQUIRE(pool && desc && out_idx && out_col && out_mask && out_rel_pos && out_rel_dist, "se3_knn_rows_paged_bucket_fwd: null pointer");
  SE3_REQUIRE(num_clouds > 0 && rows >= num_clouds, "se3_knn_rows_paged_bucket_fwd: need 0 < num_clouds <= rows (got %d clouds, %d rows)",
              num_clouds, rows);
  SE3_REQUIRE(page_size >= 1, "se3_knn_rows_paged_bucket_fwd: page_size must be >= 1 (got %d)", page_size);
  SE3_REQUIRE(n_max > 1, "se3_knn_rows_paged_bucket_fwd: need n_max > 1 (got %d)", n_max);
  SE3_REQUIRE(K >= 1 && K <= KNN_TILE, "se3_knn_rows_paged_bucket_fwd: K must be in [1, %d] (got %d)", KNN_TILE, K);
  const int B = num_clouds;
  return launch_knn_rows_paged<true>(pool, reinterpret_cast<const int*>(desc + 5 * B + 1), neighbor_mask, desc, desc + B + 1,
                                     desc + 2 * B + 1, desc + 3 * B + 1, desc + 4 * B + 1, B, rows, page_size, n_max, K, valid_radius,
                                     causal, out_idx, out_col, out_mask, out_rel_pos, out_rel_dist, stream);
}

extern "C" int se3_pair_lookup_fwd(const int64_t* row_ptr, const int* cols, int64_t nnz, int64_t batch_stride, const int64_t* idx,
                                   int b, int n, int k, int64_t* out, void* stream) {
  using namespace se3;
  SE3_REQUIRE(b > 0 && n > 0 && k > 0 && nnz >= 0, "se3_pair_lookup_fwd: bad sizes (b=%d n=%d k=%d nnz=%lld)", b, n, k,
              (long long)nnz);
  SE3_REQUIRE(batch_stride == 0 || batch_stride == n, "se3_pair_lookup_fwd: batch stride must be 0 or n");
  const int64_t total = (int64_t)b * n * k;
  const int threads = 256;
  pair_lookup_kernel<<<(unsigned)ceil_div(total, threads), threads, 0, as_stream(stream)>>>(row_ptr, cols, nnz, batch_stride, idx, n,
                                                                                            k, total, out);
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
