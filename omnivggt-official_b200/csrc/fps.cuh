// Farthest point sampling (po_utils/misc.py:114-148, farthest_point_sample): one persistent launch per call.
//
// Every step of a batch updates the running distance of each point to the last sample, then finds the point with the
// largest distance, lowest index among ties.  Distances lie in [+0, 1e10] (a NaN or a d2 above 1e10 never updates them), so
// their fp32 bits order as unsigned integers and the winner is the max of one 64-bit key (bits(dist) << 32) | ~index: no
// float atomics, and the result does not depend on how the points are split over threads or CTAs.
//
// Two kernels share the step body (fps_cta_step):
//   - fps_cta_kernel: one CTA per batch with every point in shared memory, N <= FPS_CTA_POINTS.  One __syncthreads per step.
//   - fps_grid_kernel: a cooperative launch, the grid split into groups of G CTAs, one group per batch at a time.  Each CTA holds
//     up to FPS_CTA_POINTS of its chunk in shared memory and streams the rest from global memory (L2).  Per step a CTA publishes
//     its winner (key and coordinates) in a ring of two per-CTA slots, arrives on its batch's counter with release semantics, and
//     waits with acquire loads until all G CTAs of the group have arrived; then warp 0 reduces the G slots.  The counter only
//     grows, so nothing is reset within a call.
#pragma once

#include <cuda_runtime.h>

namespace ovg {

constexpr int FPS_THREADS = 1024;
constexpr int FPS_WARPS = FPS_THREADS / 32;
constexpr int FPS_CTA_POINTS = OVG_FPS_CTA_POINTS;       // points a CTA holds in shared memory: 14336 x 16 B = 224 KB
constexpr int FPS_SMEM_BYTES = FPS_CTA_POINTS * 16;
constexpr int FPS_MAX_CTAS = 1024;                       // winner slots per ring entry
static_assert(FPS_WARPS == 32, "the block reduction reads one partial per lane");

struct FpsSlot {                                         // a CTA's winner of one step
  unsigned long long key;
  float x, y, z, pad;
};

struct FpsParams {
  const float* xyz;             // [B][N][3]
  const long long* start;       // [B] first index of each batch (device)
  long long* inds;              // [B][npoint]
  float* dist;                  // [B][N] running distances of the streamed points (grid path)
  unsigned* arrive;             // [B] arrivals per batch, zero at launch (grid path)
  FpsSlot* slots;               // [2][FPS_MAX_CTAS] (grid path)
  long long N;
  int B, npoint, ends;
  int G, groups;                // grid path: CTAs per group, groups
};

__device__ __forceinline__ float fps_d2(float x, float y, float z, float cx, float cy, float cz) {
  const float dx = __fsub_rn(x, cx), dy = __fsub_rn(y, cy), dz = __fsub_rn(z, cz);
  return __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
}

// max over the warp of 64-bit keys: the largest high word, then the largest low word among the lanes that have it
__device__ __forceinline__ unsigned long long fps_warp_max(unsigned long long k) {
  const unsigned hi = __reduce_max_sync(0xffffffffu, static_cast<unsigned>(k >> 32));
  const unsigned lo = __reduce_max_sync(0xffffffffu, static_cast<unsigned>(k >> 32) == hi ? static_cast<unsigned>(k) : 0u);
  return (static_cast<unsigned long long>(hi) << 32) | lo;
}

__device__ __forceinline__ unsigned fps_ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ void fps_red_release(unsigned* p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// The first sample of a step that does not come from the previous argmax: the start, or with include_ends 0 then N-1.
__device__ __forceinline__ long long fps_forced(const FpsParams& p, int b, int i) {
  if (p.ends) return i == 0 ? 0 : p.N - 1;
  const long long s = p.start[b];
  return (s >= 0 && s < p.N) ? s : 0;                    // an out-of-range start reads point 0
}

// One CTA's part of a step: update the distances of its points to (cx, cy, cz) and return the CTA's winner key.  sp holds
// local points [0, res) as (x, y, z, dist); points [res, cnt) are read from xyz / dist at offset `base`.  Global index of
// local point j: first + j.  kStream = false: no streamed points (res == cnt).
template <bool kStream>
__device__ __forceinline__ unsigned long long fps_cta_step(float4* sp, int res, int cnt, const float* __restrict__ xyz,
                                                          float* dist, long long base, unsigned first, float cx, float cy,
                                                          float cz, unsigned long long (*part)[FPS_WARPS], int parity) {
  float best = -1.f;
  int bj = 0;
#pragma unroll 1
  for (int j = threadIdx.x; j < res; j += FPS_THREADS) {
    const float4 q = sp[j];
    const float d = fps_d2(q.x, q.y, q.z, cx, cy, cz);
    float w = q.w;
    if (d < w) {
      w = d;
      sp[j].w = d;
    }
    if (w > best) {
      best = w;
      bj = j;
    }
  }
  for (int j = res + threadIdx.x; kStream && j < cnt; j += FPS_THREADS) {
    const float* q = xyz + (base + j) * 3;
    const float d = fps_d2(__ldg(q), __ldg(q + 1), __ldg(q + 2), cx, cy, cz);
    float w = dist[base + j];
    if (d < w) {
      w = d;
      dist[base + j] = d;
    }
    if (w > best) {
      best = w;
      bj = j;
    }
  }
  const unsigned long long key =
      best < 0.f ? 0ull : (static_cast<unsigned long long>(__float_as_uint(best)) << 32) | ~(first + static_cast<unsigned>(bj));
  const unsigned long long k = fps_warp_max(key);
  if ((threadIdx.x & 31) == 0) part[parity][threadIdx.x >> 5] = k;
  __syncthreads();
  return fps_warp_max(part[parity][threadIdx.x & 31]);   // every warp reduces the partials: no second barrier
}

// Loads local points [0, res) into shared memory and sets the distances of [res, cnt) in global memory to 1e10.
__device__ __forceinline__ void fps_load(float4* sp, int res, int cnt, const float* __restrict__ xyz, float* dist,
                                         long long base) {
  for (int j = threadIdx.x; j < res; j += FPS_THREADS) {
    const float* q = xyz + (base + j) * 3;
    sp[j] = make_float4(__ldg(q), __ldg(q + 1), __ldg(q + 2), 1e10f);
  }
  for (int j = res + threadIdx.x; j < cnt; j += FPS_THREADS) dist[base + j] = 1e10f;
}

__global__ void __launch_bounds__(FPS_THREADS, 1) fps_cta_kernel(FpsParams p) {
  extern __shared__ float4 sp[];
  __shared__ unsigned long long part[2][FPS_WARPS];
  const int b = blockIdx.x;
  const int n = static_cast<int>(p.N);
  const long long base = static_cast<long long>(b) * p.N;
  fps_load(sp, n, n, p.xyz, nullptr, base);
  __syncthreads();
  long long f = 0;
  float cx = 0.f, cy = 0.f, cz = 0.f;
  for (int i = 0; i < p.npoint; ++i) {
    if (i == 0 || (p.ends && i == 1)) f = fps_forced(p, b, i);
    if (threadIdx.x == 0) p.inds[static_cast<long long>(b) * p.npoint + i] = f;
    if (i + 1 == p.npoint) break;
    cx = sp[f].x; cy = sp[f].y; cz = sp[f].z;
    const unsigned long long k = fps_cta_step<false>(sp, n, n, p.xyz, nullptr, base, 0u, cx, cy, cz, part, i & 1);
    f = ~static_cast<unsigned>(k);
  }
}

__global__ void __launch_bounds__(FPS_THREADS, 1) fps_grid_kernel(FpsParams p) {
  extern __shared__ float4 sp[];
  __shared__ unsigned long long part[2][FPS_WARPS];
  __shared__ FpsSlot win[2];
  const int group = blockIdx.x / p.G, rank = blockIdx.x % p.G;
  if (group >= p.groups) return;                        // CTAs beyond groups * G take no part in any barrier
  const int lane = threadIdx.x & 31;
  const long long chunk = (p.N + p.G - 1) / p.G;
  const long long lo = rank * chunk;
  const int cnt = static_cast<int>(lo < p.N ? (p.N - lo < chunk ? p.N - lo : chunk) : 0);
  const int res = cnt < FPS_CTA_POINTS ? cnt : FPS_CTA_POINTS;
  const FpsSlot* mine = p.slots + group * p.G;          // this group's slots in ring entry 0
  int step = 0;                                         // steps of this CTA over all its batches: the ring parity
  for (int b = group; b < p.B; b += p.groups) {
    const long long base = static_cast<long long>(b) * p.N + lo;
    __syncthreads();                                    // the previous batch's last reads of sp are done
    fps_load(sp, res, cnt, p.xyz, p.dist, base);
    __syncthreads();
    long long f = 0;
    float cx = 0.f, cy = 0.f, cz = 0.f;
    for (int i = 0; i < p.npoint; ++i, ++step) {
      const int parity = step & 1;
      if (i == 0 || (p.ends && i == 1)) {
        f = fps_forced(p, b, i);
        const float* q = p.xyz + (static_cast<long long>(b) * p.N + f) * 3;
        cx = __ldg(q); cy = __ldg(q + 1); cz = __ldg(q + 2);
      }
      if (rank == 0 && threadIdx.x == 0) p.inds[static_cast<long long>(b) * p.npoint + i] = f;
      if (i + 1 == p.npoint) break;
      const unsigned long long k = fps_cta_step<true>(sp, res, cnt, p.xyz, p.dist, base, static_cast<unsigned>(lo), cx, cy, cz, part,
                                                parity);
      if (threadIdx.x < 32) {
        if (lane == 0) {
          FpsSlot s{k, 0.f, 0.f, 0.f, 0.f};
          if (k) {
            const int j = static_cast<int>(~static_cast<unsigned>(k) - static_cast<unsigned>(lo));
            if (j < res) {
              s.x = sp[j].x; s.y = sp[j].y; s.z = sp[j].z;
            } else {
              const float* q = p.xyz + (base + j) * 3;
              s.x = __ldg(q); s.y = __ldg(q + 1); s.z = __ldg(q + 2);
            }
          }
          p.slots[parity * FPS_MAX_CTAS + blockIdx.x] = s;
          fps_red_release(p.arrive + b, 1u);            // orders the slot store before the arrival
        }
        const unsigned target = static_cast<unsigned>(p.G) * static_cast<unsigned>(i + 1);
        while (static_cast<int>(fps_ld_acquire(p.arrive + b) - target) < 0) {
        }
        unsigned long long bk = 0;
        float bx = 0.f, by = 0.f, bz = 0.f;
        for (int r = lane; r < p.G; r += 32) {
          const FpsSlot* s = mine + parity * FPS_MAX_CTAS + r;
          const unsigned long long sk = __ldcg(&s->key);
          if (sk > bk) {
            bk = sk; bx = __ldcg(&s->x); by = __ldcg(&s->y); bz = __ldcg(&s->z);
          }
        }
        const unsigned long long wk = fps_warp_max(bk);
        const unsigned src = __ffs(__ballot_sync(0xffffffffu, bk == wk)) - 1;
        bx = __shfl_sync(0xffffffffu, bx, src);
        by = __shfl_sync(0xffffffffu, by, src);
        bz = __shfl_sync(0xffffffffu, bz, src);
        if (lane == 0) win[parity] = FpsSlot{wk, bx, by, bz, 0.f};
      }
      __syncthreads();
      f = static_cast<long long>(~static_cast<unsigned>(win[parity].key));
      cx = win[parity].x; cy = win[parity].y; cz = win[parity].z;
    }
  }
}

}  // namespace ovg
