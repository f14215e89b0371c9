// Ordered stream compaction, shared by the point cloud, the mesh, the matches and the tracks: kept items land in the order of numpy's
// boolean indexing and no atomic ever decides an output slot, so runs are bit-identical.  Block b of a count / gather kernel
// owns the tile [b COMPACT_TILE, (b + 1) COMPACT_TILE) of its items, walked in COMPACT_ITERS chunks of COMPACT_THREADS
// consecutive items.  The count kernel stores the tile's kept count (tile_sum), a scan turns the counts into tile offsets
// (block_exclusive_scan, tile_scan_kernel), and the gather kernel places each kept item at its tile offset plus its rank
// inside the tile (chunk_ranks).  The kernels keep their own predicates and emit code; these are the shared pieces.
#pragma once

namespace ovg {

constexpr int COMPACT_THREADS = 256;
constexpr int COMPACT_ITERS = 16;
constexpr int COMPACT_TILE = COMPACT_THREADS * COMPACT_ITERS;

__host__ __device__ inline long long compact_tiles(long long n) { return (n + COMPACT_TILE - 1) / COMPACT_TILE; }

// Block sum of S per-thread counts: thread s < S returns the block's total of stream s, the other threads 0.
template <int S>
__device__ __forceinline__ unsigned int tile_sum(unsigned int (&c)[S]) {
  __shared__ unsigned int warp_sum[S][COMPACT_THREADS / 32];
#pragma unroll
  for (int s = 0; s < S; ++s) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) c[s] += __shfl_xor_sync(0xffffffffu, c[s], o);
    if ((threadIdx.x & 31) == 0) warp_sum[s][threadIdx.x >> 5] = c[s];
  }
  __syncthreads();
  unsigned int sum = 0;
  if (threadIdx.x < S) {
#pragma unroll
    for (int w = 0; w < COMPACT_THREADS / 32; ++w) sum += warp_sum[threadIdx.x][w];
  }
  return sum;
}

// Ranks of a chunk of COMPACT_THREADS items in S streams: rank[s] = the set flags of stream s before this thread in the chunk,
// sum[s] = the chunk's set flags.  Ballot / popc within a warp, a scan over the warps.
template <int S>
__device__ __forceinline__ void chunk_ranks(const bool (&flag)[S], unsigned int (&rank)[S], unsigned int (&sum)[S]) {
  __shared__ unsigned int pre[S][COMPACT_THREADS / 32 + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned int ballot[S];
#pragma unroll
  for (int s = 0; s < S; ++s) {
    ballot[s] = __ballot_sync(0xffffffffu, flag[s]);
    if (lane == 0) pre[s][warp + 1] = __popc(ballot[s]);
  }
  __syncthreads();
  if (threadIdx.x < S) {
    pre[threadIdx.x][0] = 0;
#pragma unroll
    for (int w = 1; w <= COMPACT_THREADS / 32; ++w) pre[threadIdx.x][w] += pre[threadIdx.x][w - 1];
  }
  __syncthreads();
#pragma unroll
  for (int s = 0; s < S; ++s) {
    rank[s] = pre[s][warp] + __popc(ballot[s] & ((1u << lane) - 1u));
    sum[s] = pre[s][COMPACT_THREADS / 32];
  }
  __syncthreads();                                 // pre is rewritten by the next chunk
}

// chunk_ranks for per-thread counts instead of flags: rank[s] = the sum of val[s] over the threads before this one in the
// chunk, sum[s] = the chunk's total.  An inclusive shuffle scan within a warp, a scan over the warps.
template <int S>
__device__ __forceinline__ void chunk_sums(const unsigned int (&val)[S], unsigned int (&rank)[S], unsigned int (&sum)[S]) {
  __shared__ unsigned int pre[S][COMPACT_THREADS / 32 + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  unsigned int inc[S];
#pragma unroll
  for (int s = 0; s < S; ++s) {
    inc[s] = val[s];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned int t = __shfl_up_sync(0xffffffffu, inc[s], o);
      if (lane >= o) inc[s] += t;
    }
    if (lane == 31) pre[s][warp + 1] = inc[s];
  }
  __syncthreads();
  if (threadIdx.x < S) {
    pre[threadIdx.x][0] = 0;
#pragma unroll
    for (int w = 1; w <= COMPACT_THREADS / 32; ++w) pre[threadIdx.x][w] += pre[threadIdx.x][w - 1];
  }
  __syncthreads();
#pragma unroll
  for (int s = 0; s < S; ++s) {
    rank[s] = pre[s][warp] + inc[s] - val[s];
    sum[s] = pre[s][COMPACT_THREADS / 32];
  }
  __syncthreads();
}

// One block of 1024 threads: exclusive scan of cnt[0, len) into out (out may be cnt when Tin is Tout), runs per thread,
// Hillis-Steele over the runs; returns the total to every thread.
template <typename Tin, typename Tout>
__device__ Tout block_exclusive_scan(const Tin* cnt, Tout* out, long long len) {
  __shared__ Tout run[1024];
  const long long per = (len + 1023) / 1024;
  const long long c0 = threadIdx.x * per, c1 = min(c0 + per, len);
  Tout s = 0;
  for (long long c = c0; c < c1; ++c) s += cnt[c];
  run[threadIdx.x] = s;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {
    const Tout t = threadIdx.x >= o ? run[threadIdx.x - o] : Tout(0);
    __syncthreads();
    run[threadIdx.x] += t;
    __syncthreads();
  }
  Tout off = run[threadIdx.x] - s;
  for (long long c = c0; c < c1; ++c) {
    const Tout x = cnt[c];
    out[c] = off;
    off += x;
  }
  const Tout total = run[1023];
  __syncthreads();
  return total;
}

// One block of 1024 threads: offset = exclusive scan of the n tile counts, *total = their sum.
__global__ void __launch_bounds__(1024) tile_scan_kernel(const unsigned int* count, unsigned long long* offset,
                                                         unsigned long long* total, long long n) {
  const unsigned long long t = block_exclusive_scan(count, offset, n);
  if (threadIdx.x == 0) *total = t;
}

}  // namespace ovg
