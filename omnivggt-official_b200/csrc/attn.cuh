// Fused softmax(Q K^T) V for head_dim 64, non-causal, ragged sequence length (sm_90a, wgmma + TMA).
// Replaces F.scaled_dot_product_attention at reference layers/attention.py:61-66 for both the frame-wise
// (batch = B*S, N = 1374) and the global (batch = B, N = S*1374) attention of models/aggregator.py:312-341.
//
// q is pre-scaled by (1/sqrt(64))*log2(e) in the QKV GEMM epilogue, so probabilities are exp2(s - m).
// Online softmax with a running row maximum; S, P and O stay in registers (P is the A operand of the PV wgmma).
#pragma once
#include "ptx.cuh"

namespace ovg {

struct AttnParams {
  int n;        // number of query rows per (batch, head)
  int nkv;      // number of keys / values per (batch, head); == n for self-attention over one buffer
  int heads;
  int C;        // heads * 64 (row stride of `out`)
  __nv_bfloat16* out;  // [batch, n, C]
  int q_tiles;         // ceil(n / 128)
  int items;           // work items: (batch, head, q tile) tiles -- item = bh * q_tiles + q tile -- walked by the persistent grid, or,
                       // with parts > 1 (one CTA per item), n_full whole tiles followed by the LAST tiles cut into `parts` KV ranges
  int n_full, parts;   // parts <= 1: no split
  float* part_o;       // [(tile - n_full) * parts + part][128][64] un-normalised O of a KV range
  float2* part_ml;     // ... [128] (softmax reference, row sum) of that range; attn_merge_kernel combines them
};

constexpr int ATT_TILE_BYTES = 128 * 64 * 2;

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// CTA = 128 query rows of one (batch, head), 384 threads, one CTA per SM (~112 KB smem):
//   warpgroup 0: TMA producer (one thread) -- Q once per work item, K / V tiles of 128 keys through a 3-stage ring;
//   warpgroups 1, 2: 64 query rows each -- S = Q K^T (wgmma, 64 x 128 fp32 in registers), softmax, O += P V (wgmma with P
//   from registers, V MN-major from smem).  Each warpgroup waits for its own MMAs before its softmax (wgmma_wait<0> after
//   S and after P V), and nothing schedules the two warpgroups against each other: any overlap of one's softmax with the
//   other's MMAs is incidental.  Known limit: this reaches about a third of the data-sheet bf16 rate on the global attention
//   (DESIGN.md, "Measurement"); an enforced ping-pong between the warpgroups and issuing S(j+1) before the softmax of step j
//   are the next steps.
constexpr int ATT1_THREADS = 384;
constexpr int ATT1_KV_STAGES = 3;
constexpr int ATT1_SMEM_BYTES = (1 + 2 * ATT1_KV_STAGES) * ATT_TILE_BYTES + 1024 + 256;

__global__ void __launch_bounds__(ATT1_THREADS, 1)
attn1_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
             const __grid_constant__ CUtensorMap tmV, const AttnParams p) {
  constexpr int NS = ATT1_KV_STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = smem + ATT_TILE_BYTES;
  uint8_t* sV = sK + NS * ATT_TILE_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + NS * ATT_TILE_BYTES);
  uint64_t* q_full = bars;             // [1]
  uint64_t* q_empty = bars + 1;        // [1] both consumer warpgroups have finished their last S MMA of the item
  uint64_t* k_full = bars + 2;         // [NS]
  uint64_t* k_empty = k_full + NS;     // [NS]
  uint64_t* v_full = k_empty + NS;     // [NS]
  uint64_t* v_empty = v_full + NS;     // [NS]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // KV tile range [jb, jb + nkv) of this CTA's work items: everything, or -- tail tiles of a long sequence, one CTA per item --
  // one of `parts` ranges whose partial results attn_merge_kernel combines (fills the last, partly empty wave of CTAs).
  const bool is_part = p.parts > 1 && static_cast<int>(blockIdx.x) >= p.n_full;
  auto part_of = [&]() { const int i = blockIdx.x - p.n_full; return i - (i / p.parts) * p.parts; };
  auto split_tile_of = [&]() { return p.n_full + static_cast<int>(blockIdx.x - p.n_full) / p.parts; };
  int nkv = (p.nkv + 127) / 128, jb = 0;
  if (is_part) {
    const int part = part_of();
    jb = part * nkv / p.parts;
    nkv = (part + 1) * nkv / p.parts - jb;
  }

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmQ);
    tma_prefetch_desc(&tmK);
    tma_prefetch_desc(&tmV);
    mbar_init(q_full, 1);
    mbar_init(q_empty, 8);             // one arrive per consumer warp
    for (int i = 0; i < NS; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&k_empty[i], 8);
      mbar_init(&v_full[i], 1);
      mbar_init(&v_empty[i], 8);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    reg_dealloc<24>();
    if (threadIdx.x == 0) {
      int s = 0;
      uint32_t ph = 0, iph = 0;
      for (int item = blockIdx.x; item < p.items; item += gridDim.x, iph ^= 1) {
        const int tile = is_part ? split_tile_of() : item;
        const int bh = tile / p.q_tiles, q0 = (tile - bh * p.q_tiles) * 128;
        mbar_wait_quiet(q_empty, iph ^ 1);          // (first item: passes) the previous item's last S MMAs have completed
        mbar_expect_tx(q_full, ATT_TILE_BYTES);
        tma_load_3d(sQ, &tmQ, q_full, 0, q0, bh);
        for (int j = 0; j < nkv; ++j) {
          mbar_wait_quiet(&k_empty[s], ph ^ 1);
          mbar_expect_tx(&k_full[s], ATT_TILE_BYTES);
          tma_load_3d(sK + s * ATT_TILE_BYTES, &tmK, &k_full[s], 0, (jb + j) * 128, bh);
          mbar_wait_quiet(&v_empty[s], ph ^ 1);
          mbar_expect_tx(&v_full[s], ATT_TILE_BYTES);
          tma_load_3d(sV + s * ATT_TILE_BYTES, &tmV, &v_full[s], 0, (jb + j) * 128, bh);
          if (++s == NS) {
            s = 0;
            ph ^= 1;
          }
        }
      }
    }
  } else {
    reg_alloc<240>();
    const int cw = (warp >> 2) - 1;                       // consumer warpgroup: query rows [64 cw, 64 cw + 64) of the tile
    const int row0 = cw * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's rows: row0, row0 + 8
    const int fcol = 2 * (lane & 3);                      // and columns 8 j + fcol, + 1 of every accumulator
    const uint64_t qdesc = make_sw128_desc(smem_u32(sQ + cw * 64 * 128));
    int s = 0;
    uint32_t ph = 0, iph = 0;
    for (int item = blockIdx.x; item < p.items; item += gridDim.x, iph ^= 1) {
      const int tile = is_part ? split_tile_of() : item;
      const int bh = tile / p.q_tiles;
      const int q0 = (tile - bh * p.q_tiles) * 128;
      const int kv_rem = p.nkv - jb * 128;           // keys from this item's first KV tile to the end of the sequence
      float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
      float o[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] = 0.f;
      mbar_wait_quiet(q_full, iph);
      for (int j = 0; j < nkv; ++j) {
        const int kv_valid = min(128, kv_rem - j * 128);
        float sc[64];
        mbar_wait_quiet(&k_full[s], ph);
        const uint64_t kdesc = make_sw128_desc(smem_u32(sK + s * ATT_TILE_BYTES));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_ss<128, false>(sc, qdesc + 2 * k, kdesc + 2 * k, k > 0);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs<64>(sc);
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&k_empty[s]);
          if (j + 1 == nkv) mbar_arrive(q_empty);
        }
        if (kv_valid < 128) {
#pragma unroll
          for (int i = 0; i < 64; ++i)
            if (8 * (i >> 2) + fcol + (i & 1) >= kv_valid) sc[i] = -INFINITY;
        }
        // online softmax: row maxima over the quad of threads that share a row
        float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
        for (int i = 0; i < 64; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], sc[i]);
        float alpha[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
          mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
          const float m_new = fmaxf(m_run[h], mx[h]);
          alpha[h] = ex2_approx(m_run[h] - m_new);         // first tile: exp2(-inf) = 0
          m_run[h] = m_new;
          l_run[h] *= alpha[h];
        }
        uint32_t pa[32];                                  // P as bf16 A fragments: 8 k-steps of 16 keys x 4 registers
#pragma unroll
        for (int i = 0; i < 64; i += 2) {
          const int h = (i >> 1) & 1;
          const float e0 = ex2_approx(sc[i] - m_run[h]), e1 = ex2_approx(sc[i + 1] - m_run[h]);
          l_run[h] += e0 + e1;
          pa[i >> 1] = pack_bf16(e0, e1);
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) o[i] *= alpha[(i >> 1) & 1];
        mbar_wait_quiet(&v_full[s], ph);
        const uint64_t vdesc = make_sw128_desc(smem_u32(sV + s * ATT_TILE_BYTES));
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) wgmma_rs64_bf16_tb(o, pa + 4 * kk, vdesc + static_cast<uint64_t>(kk) * (2048 >> 4), 1);
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs<32>(o);
        __syncwarp();
        if (lane == 0) mbar_arrive(&v_empty[s]);
        if (++s == NS) {
          s = 0;
          ph ^= 1;
        }
      }
      // ---- epilogue: O / l -> bf16 -> out[b, qrow, head*64 .. +64)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 1);
        l_run[h] += __shfl_xor_sync(0xffffffffu, l_run[h], 2);
      }
      const int head = bh % p.heads, bz = bh / p.heads;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = row0 + 8 * h;
        if (is_part) {     // one KV range of a split tile: un-normalised O, reference and row sum for attn_merge_kernel
          const long long sidx = static_cast<long long>(blockIdx.x) - p.n_full;     // == (tile - n_full) * parts + part
          float* dst = p.part_o + (sidx * 128 + r) * 64 + fcol;
#pragma unroll
          for (int j = 0; j < 8; ++j) *reinterpret_cast<float2*>(dst + 8 * j) = make_float2(o[4 * j + 2 * h], o[4 * j + 2 * h + 1]);
          if ((lane & 3) == 0) p.part_ml[sidx * 128 + r] = make_float2(m_run[h], l_run[h]);
        } else if (q0 + r < p.n) {
          const float inv = 1.0f / l_run[h];
          __nv_bfloat16* dst = p.out + (static_cast<long long>(bz) * p.n + q0 + r) * p.C + head * 64 + fcol;
#pragma unroll
          for (int j = 0; j < 8; ++j)
            *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16(o[4 * j + 2 * h] * inv, o[4 * j + 2 * h + 1] * inv);
        }
      }
    }
  }
}

// Combine the KV ranges of the split tiles: out = sum_i 2^(m_i - M) O_i / sum_i 2^(m_i - M) l_i, M = max_i m_i (fixed order of the
// parts: deterministic).  One block per split tile, one thread per query row.
__global__ void __launch_bounds__(128) attn_merge_kernel(const AttnParams p) {
  const int tile = p.n_full + blockIdx.x, r = threadIdx.x;
  const int bh = tile / p.q_tiles;
  const int qrow = (tile - bh * p.q_tiles) * 128 + r;
  if (qrow >= p.n) return;
  const int head = bh % p.heads, bz = bh / p.heads;
  const long long s0 = static_cast<long long>(blockIdx.x) * p.parts;
  float M = -INFINITY;
  for (int i = 0; i < p.parts; ++i) M = fmaxf(M, p.part_ml[(s0 + i) * 128 + r].x);
  float acc[64];
#pragma unroll
  for (int c = 0; c < 64; ++c) acc[c] = 0.f;
  float L = 0.f;
  for (int i = 0; i < p.parts; ++i) {
    const float2 ml = p.part_ml[(s0 + i) * 128 + r];
    const float w = exp2f(ml.x - M);
    L = fmaf(w, ml.y, L);
    const float4* o4 = reinterpret_cast<const float4*>(p.part_o + ((s0 + i) * 128 + r) * 64);
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      const float4 t = o4[c];
      acc[4 * c] = fmaf(w, t.x, acc[4 * c]);
      acc[4 * c + 1] = fmaf(w, t.y, acc[4 * c + 1]);
      acc[4 * c + 2] = fmaf(w, t.z, acc[4 * c + 2]);
      acc[4 * c + 3] = fmaf(w, t.w, acc[4 * c + 3]);
    }
  }
  const float inv = 1.0f / L;
  uint4* dst = reinterpret_cast<uint4*>(p.out + (static_cast<long long>(bz) * p.n + qrow) * p.C + head * 64);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    uint4 w;
    w.x = pack_bf16(acc[8 * i + 0] * inv, acc[8 * i + 1] * inv);
    w.y = pack_bf16(acc[8 * i + 2] * inv, acc[8 * i + 3] * inv);
    w.z = pack_bf16(acc[8 * i + 4] * inv, acc[8 * i + 5] * inv);
    w.w = pack_bf16(acc[8 * i + 6] * inv, acc[8 * i + 7] * inv);
    dst[i] = w;
  }
}

}  // namespace ovg
