// Persistent warp-specialised wgmma GEMM for sm_90a with fused epilogues.
//
//   D[M,N] = sum_taps A[m + tap_off[t], 0:Kc] * B[n, t*Kc:(t+1)*Kc]^T      (bf16 x bf16 -> fp32 in registers)
//
// One kernel serves every dense contraction on the hot path:
//   * aggregator linears  (reference layers/attention.py:52,:75, layers/mlp.py:35-38)  -- 1 tap
//   * DPT 1x1 / transposed convs (heads/dpt_head.py:69-96)                              -- 1 tap
//   * DPT 3x3 convs as 9 row-shifted GEMMs over a zero-bordered ("padded-linear") NHWC
//     layout (heads/dpt_head.py:326-354,:379-399,:115-126)                              -- 9 taps
// Roles (512 threads, setmaxnreg split 40 / 144 / 184 registers = the whole 64K register file):
//   warpgroup 0     TMA producer (one thread), 40 registers
//   warpgroups 1-2  wgmma consumers, 64 rows of the 128-row tile each; they issue MMAs and stage the accumulators, nothing else
//                   (144 registers)
//   warpgroup 3     epilogue: one whole accumulator row per thread, every column of the tile (184 registers); the residual
//                   epilogue instead walks the tile row by row across each warp, so that its fp32 read-modify-write is coalesced
// Pipeline: smem full/empty ring (TMA<->MMA).  The finished accumulator tile goes through ONE fp32 smem tile (sAcc) so that
// the epilogue works on whole rows, as the QKV head LayerNorm and the row remaps need.  Hand-off over two named barriers of
// the 384 consumer + epilogue threads: the consumers wait for GEMM_BAR_ACC_FREE (skipped on their first tile), store the
// accumulators and arrive on GEMM_BAR_ACC_FULL; the epilogue waits for GEMM_BAR_ACC_FULL, runs the fused epilogue and arrives on
// GEMM_BAR_ACC_FREE (not after its last tile, so that both barriers end balanced).  The epilogue of tile i thus runs under
// the MMAs of tile i + 1; the consumers stall only when an epilogue takes longer than a K loop.
#pragma once
#include "ptx.cuh"

namespace ovg {

enum EpiKind { EPI_BF16 = 0, EPI_RESID = 1, EPI_QKV = 2, EPI_HEADTAIL = 3 };
enum RowMap { RM_IDENT = 0, RM_DENSE2PAD = 1, RM_PAD = 2, RM_PIXSHUF = 3 };

struct GemmParams {
  int M, N;
  int k_blocks;    // total 64-wide K blocks
  int kc_blocks;   // K blocks per tap
  int tap_off[9];  // A row offset of each tap
  // ---- common epilogue
  const float* bias;  // [N] ([cout] for RM_PIXSHUF) or nullptr
  int act;            // 0 none, 1 exact-erf GELU, 2 ReLU
  void* out;
  long long ldo;  // elements
  // ---- EPI_BF16
  const float* table;  // additive fp32 [table_rows][N] indexed by (m % table_rows), or nullptr
  int table_rows;
  int f16;                     // EPI_BF16 / EPI_HEADTAIL: operands, skips and the 16-bit output are IEEE half instead of bf16
  const __nv_bfloat16* skip1;  // optional addends, indexed like `out`
  const __nv_bfloat16* skip2;
  int rowmap;  // RowMap
  int gh, gw;  // source grid (rows are (frame, y, x)); RM_PAD: interior size of the padded domain
  int ps, cout;  // RM_PIXSHUF: stride (= kernel) and output channels
  // ---- EPI_RESID (epilogue_resid_tile):  out(fp32)[row,n] += gamma[n] * (acc + bias[n]),  row = row_index ? row_index[m] : m
  const float* gamma;
  const int* row_index;
  // ---- EPI_QKV (layers/attention.py:52-58 fused: bias, q/k LayerNorm(64), 2-D RoPE, head-major bf16)
  __nv_bfloat16* q_out;
  __nv_bfloat16* k_out;
  __nv_bfloat16* v_out;
  int C, ntok, T, nspecial, wp, maxpos;
  const float* qn_w;
  const float* qn_b;
  const float* kn_w;
  const float* kn_b;
  const float* rope_cos;  // [maxpos][16]
  const float* rope_sin;
  float qscale;  // softmax scale * log2(e), folded into q
  int qk_norm;   // 1: LayerNorm(64) on q,k (aggregator blocks); 0: plain (DINOv2 blocks)
  int rope;      // 1: 2-D RoPE on q,k
  // context parallelism: K and V rows of this rank's tokens are stored into every rank's full-length K / V buffer
  // ([batch*heads, peer_ntok, 64], this rank's tokens starting at row peer_tok_off) instead of k_out / v_out
  __nv_bfloat16* k_peer[8];
  __nv_bfloat16* v_peer[8];
  int n_peers;
  int peer_ntok;
  long long peer_tok_off;
  // ---- EPI_HEADTAIL (heads/dpt_head.py:121-126 + heads/head_act.py:61-112): relu, 1x1 32->outc, activation
  const float* w2;  // [outc][32]
  const float* b2;  // [outc]
  int outc;         // 2 (depth) or 4 (points)
  int head_act;     // 0 exp, 1 inverse-log
  float* preds;     // [F,gh,gw,outc-1]
  float* conf;      // [F,gh,gw]
};

constexpr int GEMM_BM = 128;
constexpr int GEMM_BK = 64;
constexpr int GEMM_THREADS = 512;
constexpr int GEMM_EPI_THREAD0 = 384;     // first thread of the epilogue warpgroup
constexpr int GEMM_BAR_ACC_FULL = 1;      // named barriers over the 256 consumer + 128 epilogue threads
constexpr int GEMM_BAR_ACC_FREE = 2;
// setmaxnreg split; the three warpgroups share the 64K-entry register file.  The QKV epilogue (two 64-wide heads per row at
// BN = 128) needs the most: it spills at 168.  The wgmma warpgroups hold BN / 2 accumulators and little else.
constexpr int GEMM_PRODUCER_REGS = 40;
constexpr int GEMM_MMA_REGS = 144;
constexpr int GEMM_EPI_REGS = 184;
static_assert(128 * (GEMM_PRODUCER_REGS + 2 * GEMM_MMA_REGS + GEMM_EPI_REGS) <= 65536, "register split");
constexpr int GEMM_A_BYTES = GEMM_BM * GEMM_BK * 2;

constexpr int GEMM_QKV_TABLE_BYTES = 3 * 64 * 18 * 4 + 1024;   // QKV epilogue: rope cos / sin / -sin + q,k LayerNorm affine
// BN <= 128: a 128 x 256 tile would need 128 accumulator registers per thread plus a 128 KB fp32 smem tile, which leaves room
// for only two K stages within the 227 KB of an H100 SM.
template <int BN>
struct GemmCfg {
  static_assert(BN == 32 || BN == 64 || BN == 128, "block_n");
  static constexpr int B_BYTES = BN * GEMM_BK * 2;
  static constexpr int STAGE_BYTES = GEMM_A_BYTES + B_BYTES;
  static constexpr int STAGES = BN >= 128 ? 4 : 6;
  static constexpr int ACC_LD = BN + 4;   // fp32 row pitch of the accumulator tile: row-wise float4 reads are conflict-free
  static constexpr int ACC_BYTES = GEMM_BM * ACC_LD * 4;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + ACC_BYTES + 1024 /*align*/ + 256 /*barriers*/ + GEMM_QKV_TABLE_BYTES;
};

// Exact-erf GELU (nn.GELU() default, reference layers/mlp.py:22,:36) with erf evaluated by Abramowitz-Stegun 7.1.26
// (|abs err| <= 1.5e-7, three orders below the bf16 output resolution): 2 MUFU (rcp, ex2) + FMA-pipe work per element;
// erff() costs ~3x more and made the fc1 epilogue longer than its K = 1024 mainloop.
__device__ __forceinline__ float2 gelu_erf2(const float2 x) {
  const float2 z = make_float2(fabsf(x.x) * 0.70710678118654752f, fabsf(x.y) * 0.70710678118654752f);
  const float2 d = ffma2(make_float2(0.3275911f, 0.3275911f), z, make_float2(1.0f, 1.0f));
  float2 t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t.x) : "f"(d.x));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t.y) : "f"(d.y));
  float2 poly = ffma2(make_float2(1.061405429f, 1.061405429f), t, make_float2(-1.453152027f, -1.453152027f));
  poly = ffma2(poly, t, make_float2(1.421413741f, 1.421413741f));
  poly = ffma2(poly, t, make_float2(-0.284496736f, -0.284496736f));
  poly = ffma2(poly, t, make_float2(0.254829592f, 0.254829592f));
  poly = fmul2(poly, t);
  const float2 a = fmul2(fmul2(z, make_float2(-1.4426950408889634f, -1.4426950408889634f)), z);
  float2 e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.x) : "f"(a.x));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e.y) : "f"(a.y));
  // erf_abs = 1 - poly * e;  gelu = 0.5 x (1 + sign(x) erf_abs) = 0.5 x + (0.5 |x|) (1 - poly e)
  const float2 hx = fmul2(x, make_float2(0.5f, 0.5f));
  const float2 hax = fmul2(z, make_float2(0.70710678118654752f, 0.70710678118654752f));   // 0.5 |x|
  const float2 w = ffma2(fmul2(poly, e), make_float2(-1.0f, -1.0f), make_float2(1.0f, 1.0f));
  return ffma2(hax, w, hx);
}

// 32 consecutive fp32 accumulator values of this thread's row (16-byte aligned smem)
__device__ __forceinline__ void acc_ld32(const float* src, uint32_t* r) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 v = reinterpret_cast<const float4*>(src)[i];
    r[4 * i] = __float_as_uint(v.x); r[4 * i + 1] = __float_as_uint(v.y);
    r[4 * i + 2] = __float_as_uint(v.z); r[4 * i + 3] = __float_as_uint(v.w);
  }
}

// One 128 x BN accumulator tile: smem -> registers -> fused epilogue -> global.  `arow` is this thread's row of the fp32
// accumulator tile, `m` its global row; this thread owns every column of the row.
template <int BN, int EPI>
__device__ __forceinline__ void epilogue_tile(const GemmParams& p, const float* arow, const int m, const int n0,
                                              const float* s_rope) {
  if constexpr (EPI == EPI_QKV) {
    // ---- per-row RoPE position (reference omnivggt_aggregator.py:215-224; layers/rope.py:39-59)
    int py = 0, px = 0;
    {
      const int t = m % p.T;
      if (t >= p.nspecial) {
        const int pp = t - p.nspecial;
        py = pp / p.wp + 1;
        px = pp % p.wp + 1;
      }
    }
    // smem tables (filled at kernel start): [cos | sin | -sin][64 positions][18] (16 frequencies, rows padded to 18
    // floats so that float2 reads stay aligned), then the q / k LayerNorm affine [qw*qscale | qb*qscale | kw | kb][64].
    const float2* cy = reinterpret_cast<const float2*>(s_rope + py * 18);
    const float2* sy = reinterpret_cast<const float2*>(s_rope + 64 * 18 + py * 18);
    const float2* nsy = reinterpret_cast<const float2*>(s_rope + 128 * 18 + py * 18);
    const float2* cx = reinterpret_cast<const float2*>(s_rope + px * 18);
    const float2* sx = reinterpret_cast<const float2*>(s_rope + 64 * 18 + px * 18);
    const float2* nsx = reinterpret_cast<const float2*>(s_rope + 128 * 18 + px * 18);
    const float* s_ln = s_rope + 3 * 64 * 18;
    const long long seq = m / p.ntok;
    const long long tok = m % p.ntok;
    const int heads = p.C >> 6;
    for (int c = 0; c < BN / 64; ++c) {
      const int n = n0 + c * 64;
      if (n >= p.N) continue;                                   // warp-uniform
      if (m < p.M) {
        uint32_t raw[64];
        acc_ld32(arow + c * 64, raw);
        acc_ld32(arow + c * 64 + 32, raw + 32);
        // all arithmetic on packed fp32 pairs (FADD2 / FMUL2 / FFMA2): v2[i] = elements (2i, 2i+1) of this head
        float2 v2[32];
        {
          const float4* b4 = reinterpret_cast<const float4*>(p.bias + n);
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const float4 b = __ldg(b4 + i);
            v2[2 * i] = fadd2(make_float2(__uint_as_float(raw[4 * i + 0]), __uint_as_float(raw[4 * i + 1])), make_float2(b.x, b.y));
            v2[2 * i + 1] = fadd2(make_float2(__uint_as_float(raw[4 * i + 2]), __uint_as_float(raw[4 * i + 3])), make_float2(b.z, b.w));
          }
        }
        const int which = n / p.C;
        const int h = (n - which * p.C) >> 6;
        if (which < 2 && p.qk_norm) {
          float2 s01 = make_float2(0.f, 0.f), s23 = make_float2(0.f, 0.f);
#pragma unroll
          for (int i = 0; i < 32; i += 2) {
            s01 = fadd2(s01, v2[i]);
            s23 = fadd2(s23, v2[i + 1]);
          }
          const float mean = ((s01.x + s01.y) + (s23.x + s23.y)) * (1.0f / 64.0f);
          const float2 nm = make_float2(-mean, -mean);
          float2 q01 = make_float2(0.f, 0.f), q23 = make_float2(0.f, 0.f);
#pragma unroll
          for (int i = 0; i < 32; i += 2) {
            v2[i] = fadd2(v2[i], nm);
            v2[i + 1] = fadd2(v2[i + 1], nm);
            q01 = ffma2(v2[i], v2[i], q01);
            q23 = ffma2(v2[i + 1], v2[i + 1], q23);
          }
          const float rstd = rsqrtf(((q01.x + q01.y) + (q23.x + q23.y)) * (1.0f / 64.0f) + 1e-5f);
          const float2 rr = make_float2(rstd, rstd);
          const float4* w4 = reinterpret_cast<const float4*>(s_ln + which * 128);        // q: pre-multiplied by qscale
          const float4* b4 = reinterpret_cast<const float4*>(s_ln + which * 128 + 64);
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            const float4 w = w4[i];
            const float4 b = b4[i];
            v2[2 * i] = ffma2(fmul2(v2[2 * i], rr), make_float2(w.x, w.y), make_float2(b.x, b.y));
            v2[2 * i + 1] = ffma2(fmul2(v2[2 * i + 1], rr), make_float2(w.z, w.w), make_float2(b.z, b.w));
          }
        } else if (which == 0) {
          const float2 qs = make_float2(p.qscale, p.qscale);
#pragma unroll
          for (int i = 0; i < 32; ++i) v2[i] = fmul2(v2[i], qs);
        }
        if (which < 2 && p.rope) {
          // rotate (d, d+16) with the row angle and (32+d, 48+d) with the column angle (layers/rope.py:154-188)
#pragma unroll
          for (int k = 0; k < 8; ++k) {
            const float2 a0 = v2[k], b0 = v2[8 + k];
            v2[k] = ffma2(b0, nsy[k], fmul2(a0, cy[k]));
            v2[8 + k] = ffma2(a0, sy[k], fmul2(b0, cy[k]));
            const float2 a1 = v2[16 + k], b1 = v2[24 + k];
            v2[16 + k] = ffma2(b1, nsx[k], fmul2(a1, cx[k]));
            v2[24 + k] = ffma2(a1, sx[k], fmul2(b1, cx[k]));
          }
        }
        uint4 o8[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          o8[i].x = pack_bf16(v2[4 * i + 0].x, v2[4 * i + 0].y);
          o8[i].y = pack_bf16(v2[4 * i + 1].x, v2[4 * i + 1].y);
          o8[i].z = pack_bf16(v2[4 * i + 2].x, v2[4 * i + 2].y);
          o8[i].w = pack_bf16(v2[4 * i + 3].x, v2[4 * i + 3].y);
        }
        if (which > 0 && p.n_peers > 0) {
          // one 128-byte row per lane into every rank's buffer: plain stores over NVLink (peer-mapped memory)
          const long long roff = ((seq * heads + h) * p.peer_ntok + p.peer_tok_off + tok) * 64;
          for (int pr = 0; pr < p.n_peers; ++pr) {
            uint4* d4 = reinterpret_cast<uint4*>((which == 1 ? p.k_peer[pr] : p.v_peer[pr]) + roff);
#pragma unroll
            for (int i = 0; i < 8; ++i) d4[i] = o8[i];
          }
          continue;
        }
        uint4* d4 = reinterpret_cast<uint4*>((which == 0 ? p.q_out : (which == 1 ? p.k_out : p.v_out)) +
                                             ((seq * heads + h) * p.ntok + tok) * 64);
#pragma unroll
        for (int i = 0; i < 8; ++i) d4[i] = o8[i];
      }
    }
  } else {
    // ---- row mapping
    static_assert(EPI == EPI_BF16 || EPI == EPI_HEADTAIL, "EPI_RESID runs epilogue_resid_tile");
    const bool row_ok = m < p.M;
    bool interior = true;  // RM_PAD: border rows are written as zeros
    long long drow = m;
    int fr = 0, yy = 0, xx = 0;
    {
      if (p.rowmap == RM_DENSE2PAD || p.rowmap == RM_PIXSHUF) {
        const int hw = p.gh * p.gw;
        fr = m / hw;
        const int rem = m - fr * hw;
        yy = rem / p.gw;
        xx = rem - yy * p.gw;
        if (p.rowmap == RM_DENSE2PAD)
          drow = (static_cast<long long>(fr) * (p.gh + 2) + (yy + 1)) * (p.gw + 2) + (xx + 1);
      } else if (p.rowmap == RM_PAD) {
        const int pw = p.gw + 2;
        const int pp = (p.gh + 2) * pw;
        fr = m / pp;
        const int rem = m - fr * pp;
        yy = rem / pw;
        xx = rem - yy * pw;
        interior = (yy >= 1 && yy <= p.gh && xx >= 1 && xx <= p.gw);
      }
    }
    for (int c = 0; c < BN / 32; ++c) {
      const int n = n0 + c * 32;
      if (n >= p.N || !row_ok) continue;
      uint32_t raw[32];
      acc_ld32(arow + c * 32, raw);
      float v[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = __uint_as_float(raw[i]);

      if constexpr (EPI == EPI_HEADTAIL) {
        if (!interior) continue;
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = fmaxf(v[i] + __ldg(p.bias + i), 0.f);
        const long long pix = (static_cast<long long>(fr) * p.gh + (yy - 1)) * p.gw + (xx - 1);
        for (int o = 0; o < p.outc; ++o) {
          float acc = __ldg(p.b2 + o);
#pragma unroll
          for (int i = 0; i < 32; ++i) acc += __ldg(p.w2 + o * 32 + i) * v[i];
          if (o == p.outc - 1) {
            p.conf[pix] = 1.0f + expf(acc);
          } else {
            const float y = p.head_act == 0 ? expf(acc) : copysignf(expm1f(fabsf(acc)), acc);
            p.preds[pix * (p.outc - 1) + o] = y;
          }
        }
      } else {  // EPI_BF16
        int bn = n;      // bias / channel index
        long long dcol = n;
        if (p.rowmap == RM_PIXSHUF) {
          const int kk = n / p.cout;
          bn = n - kk * p.cout;
          const int ky = kk / p.ps, kx = kk - ky * p.ps;
          const int oh = p.gh * p.ps, ow = p.gw * p.ps;
          drow = (static_cast<long long>(fr) * (oh + 2) + (yy * p.ps + ky + 1)) * (ow + 2) + (xx * p.ps + kx + 1);
          dcol = bn;
        }
        if (p.bias) {
          const float4* b4 = reinterpret_cast<const float4*>(p.bias + bn);
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float4 b = __ldg(b4 + i);
            const float2 s01 = fadd2(make_float2(v[4 * i + 0], v[4 * i + 1]), make_float2(b.x, b.y));
            const float2 s23 = fadd2(make_float2(v[4 * i + 2], v[4 * i + 3]), make_float2(b.z, b.w));
            v[4 * i + 0] = s01.x; v[4 * i + 1] = s01.y; v[4 * i + 2] = s23.x; v[4 * i + 3] = s23.y;
          }
        }
        if (p.table) {
          const float* t = p.table + static_cast<long long>(m % p.table_rows) * p.N + n;
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] += __ldg(t + i);
        }
        const long long off = drow * p.ldo + dcol;
        if (p.skip1 && row_ok) {
          const uint4* s4 = reinterpret_cast<const uint4*>(p.skip1 + off);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const uint4 sv = __ldg(s4 + i);
            const float2 s0 = unpack_h(sv.x, p.f16), s1 = unpack_h(sv.y, p.f16), s2 = unpack_h(sv.z, p.f16), s3 = unpack_h(sv.w, p.f16);
            v[8 * i + 0] += s0.x; v[8 * i + 1] += s0.y;
            v[8 * i + 2] += s1.x; v[8 * i + 3] += s1.y;
            v[8 * i + 4] += s2.x; v[8 * i + 5] += s2.y;
            v[8 * i + 6] += s3.x; v[8 * i + 7] += s3.y;
          }
        }
        if (p.skip2 && row_ok) {
          const uint4* s4 = reinterpret_cast<const uint4*>(p.skip2 + off);
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const uint4 sv = __ldg(s4 + i);
            const float2 s0 = unpack_h(sv.x, p.f16), s1 = unpack_h(sv.y, p.f16), s2 = unpack_h(sv.z, p.f16), s3 = unpack_h(sv.w, p.f16);
            v[8 * i + 0] += s0.x; v[8 * i + 1] += s0.y;
            v[8 * i + 2] += s1.x; v[8 * i + 3] += s1.y;
            v[8 * i + 4] += s2.x; v[8 * i + 5] += s2.y;
            v[8 * i + 6] += s3.x; v[8 * i + 7] += s3.y;
          }
        }
        if (p.act == 1) {
#pragma unroll
          for (int i = 0; i < 32; i += 2) {
            const float2 g = gelu_erf2(make_float2(v[i], v[i + 1]));
            v[i] = g.x;
            v[i + 1] = g.y;
          }
        } else if (p.act == 2) {
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = fmaxf(v[i], 0.f);
        }
        if (!interior) {
#pragma unroll
          for (int i = 0; i < 32; ++i) v[i] = 0.f;
        }
        uint4* d4 = reinterpret_cast<uint4*>(reinterpret_cast<__nv_bfloat16*>(p.out) + off);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          uint4 o;
          o.x = pack_h(v[8 * i + 0], v[8 * i + 1], p.f16);
          o.y = pack_h(v[8 * i + 2], v[8 * i + 3], p.f16);
          o.z = pack_h(v[8 * i + 4], v[8 * i + 5], p.f16);
          o.w = pack_h(v[8 * i + 6], v[8 * i + 7], p.f16);
          d4[i] = o;
        }
      }
    }
  }
}

// EPI_RESID over one 128 x BN tile by the epilogue warpgroup: x[row, n] += gamma[n] * (acc + bias[n]) in fp32.  Epilogue warp
// `ew` takes rows [32 ew, 32 ew + 32); each warp access covers whole rows, BN / 4 lanes per row with one float4 each, so a row
// segment of x is one contiguous 4 * BN-byte load and store (a row per thread would touch 32 rows per access and use half of each
// 32-byte sector).  RES_INFLIGHT accesses are issued before the first is used: one warp per scheduler has to cover the HBM latency alone.
constexpr int RES_INFLIGHT = 8;
template <int BN>
__device__ __forceinline__ void epilogue_resid_tile(const GemmParams& p, const float* sAcc, const int m0, const int n0,
                                                    const int ew, const int lane) {
  constexpr int LPR = BN / 4;           // lanes per row
  constexpr int RPA = 32 / LPR;         // rows per warp access
  static_assert(32 % (RPA * RES_INFLIGHT) == 0, "rows per warp");
  const int c = 4 * (lane % LPR);
  const int n = n0 + c;
  if (n >= p.N) return;                 // N % 32 == 0: a float4 is wholly inside or outside
  const float4 g = __ldg(reinterpret_cast<const float4*>(p.gamma + n));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p.bias + n));
  for (int j0 = 0; j0 < 32; j0 += RPA * RES_INFLIGHT) {
    float4 xv[RES_INFLIGHT], a[RES_INFLIGHT];
    float* x[RES_INFLIGHT];
#pragma unroll
    for (int u = 0; u < RES_INFLIGHT; ++u) {
      const int r = 32 * ew + j0 + u * RPA + lane / LPR;
      const int m = m0 + r;
      x[u] = nullptr;
      if (m < p.M) {
        const long long drow = p.row_index ? p.row_index[m] : m;
        x[u] = reinterpret_cast<float*>(p.out) + drow * p.ldo + n;
        xv[u] = *reinterpret_cast<const float4*>(x[u]);
        a[u] = *reinterpret_cast<const float4*>(sAcc + r * GemmCfg<BN>::ACC_LD + c);
      }
    }
#pragma unroll
    for (int u = 0; u < RES_INFLIGHT; ++u) {
      if (x[u] == nullptr) continue;
      xv[u].x += g.x * (a[u].x + b.x);
      xv[u].y += g.y * (a[u].y + b.y);
      xv[u].z += g.z * (a[u].z + b.z);
      xv[u].w += g.w * (a[u].w + b.w);
      *reinterpret_cast<float4*>(x[u]) = xv[u];
    }
  }
}

// The two wgmma warpgroups of gemm_kernel: the K loop of every tile, then the accumulators into sAcc for the epilogue warpgroup.
// The operand type is a template argument, so that each K block is one straight run of wgmmas: with the choice between the bf16 and
// the fp16 form made at run time inside the loop, ptxas put a warpgroup fence in front of every wgmma and made each one wait on
// the scoreboard.
template <int BN, bool F16>
__device__ __forceinline__ void gemm_mma_loop(const GemmParams& p, uint8_t* sA, uint8_t* sB, float* sAcc, uint64_t* full,
                                              uint64_t* empty, const int num_tiles, const int warp, const int lane) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  const int cw = (warp >> 2) - 1;      // consumer warpgroup: rows [64 cw, 64 cw + 64) of the tile
  const int frow = cw * 64 + (warp & 3) * 16 + (lane >> 2);   // accumulator fragment rows frow, frow + 8
  const int fcol = 2 * (lane & 3);
  int s = 0;
  uint32_t ph = 0;
  float acc[BN / 2];
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    int prev = -1;
    for (int kb = 0; kb < p.k_blocks; ++kb) {
      mbar_wait_quiet(&full[s], ph);      // no printf call site: it would serialise the wgmma pipeline
      const uint64_t adesc = make_sw128_desc(smem_u32(sA + s * GEMM_A_BYTES + cw * 64 * 128));
      const uint64_t bdesc = make_sw128_desc(smem_u32(sB + s * Cfg::B_BYTES));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < GEMM_BK / 16; ++k) wgmma_ss<BN, F16>(acc, adesc + 2 * k, bdesc + 2 * k, (kb | k) != 0);
      wgmma_commit();
      wgmma_wait<1>();                 // the previous K block's MMAs are done: release its stage
      if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
      prev = s;
      if (++s == STAGES) {
        s = 0;
        ph ^= 1;
      }
    }
    wgmma_wait<0>();
    fence_regs<BN / 2>(acc);
    if (lane == 0) mbar_arrive(&empty[prev]);
    // the epilogue warpgroup is done with the previous tile's accumulators (it has read sAcc in full)
    if (tile != static_cast<int>(blockIdx.x)) named_sync(GEMM_BAR_ACC_FREE, 384);
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      *reinterpret_cast<float2*>(sAcc + frow * Cfg::ACC_LD + 8 * j + fcol) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(sAcc + (frow + 8) * Cfg::ACC_LD + 8 * j + fcol) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
    named_arrive(GEMM_BAR_ACC_FULL, 384);
  }
}

template <int BN, int EPI>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  using Cfg = GemmCfg<BN>;
  constexpr int STAGES = Cfg::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sA = smem;
  uint8_t* sB = smem + STAGES * GEMM_A_BYTES;
  float* sAcc = reinterpret_cast<float*>(smem + STAGES * Cfg::STAGE_BYTES);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES + Cfg::ACC_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + STAGES;
  float* s_rope = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 256);  // [3][64][18] + [4][64]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int m_tiles = (p.M + GEMM_BM - 1) / GEMM_BM;
  const int n_tiles = (p.N + BN - 1) / BN;
  const int num_tiles = m_tiles * n_tiles;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 8);     // one arrive per consumer warp
    }
    fence_barrier_init();
  }
  if (EPI == EPI_QKV && warp >= 4) {
    for (int i = threadIdx.x - 128; i < p.maxpos * 16; i += GEMM_THREADS - 128) {
      s_rope[(i >> 4) * 18 + (i & 15)] = p.rope_cos[i];
      s_rope[64 * 18 + (i >> 4) * 18 + (i & 15)] = p.rope_sin[i];
      s_rope[128 * 18 + (i >> 4) * 18 + (i & 15)] = -p.rope_sin[i];
    }
    if (p.qk_norm && threadIdx.x >= 128 && threadIdx.x < 192) {
      float* s_ln = s_rope + 3 * 64 * 18;
      const int i = threadIdx.x - 128;
      s_ln[i] = p.qn_w[i] * p.qscale;          // q is pre-scaled by log2(e)/sqrt(head_dim): fold it into the affine
      s_ln[64 + i] = p.qn_b[i] * p.qscale;
      s_ln[128 + i] = p.kn_w[i];
      s_ln[192 + i] = p.kn_b[i];
    }
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== TMA producer =====================
    reg_dealloc<GEMM_PRODUCER_REGS>();
    if (threadIdx.x == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        const int m0 = (tile / n_tiles) * GEMM_BM;
        const int n0 = (tile % n_tiles) * BN;
        for (int kb = 0; kb < p.k_blocks; ++kb) {
          mbar_wait_quiet(&empty[s], ph ^ 1);
          mbar_expect_tx(&full[s], Cfg::STAGE_BYTES);
          const int tap = kb / p.kc_blocks;
          const int c0 = (kb - tap * p.kc_blocks) * GEMM_BK;
          tma_load_2d(sA + s * GEMM_A_BYTES, &tmA, &full[s], c0, m0 + p.tap_off[tap]);
          tma_load_2d(sB + s * Cfg::B_BYTES, &tmB, &full[s], kb * GEMM_BK, n0);
          if (++s == STAGES) {
            s = 0;
            ph ^= 1;
          }
        }
      }
    }
  } else if (threadIdx.x < GEMM_EPI_THREAD0) {
    // ===================== wgmma (2 warpgroups, 8 warps) =====================
    reg_alloc<GEMM_MMA_REGS>();
    // Only EPI_BF16 / EPI_HEADTAIL take fp16 operands; the others are bf16 at compile time.
    if constexpr (EPI == EPI_BF16 || EPI == EPI_HEADTAIL) {
      if (p.f16) gemm_mma_loop<BN, true>(p, sA, sB, sAcc, full, empty, num_tiles, warp, lane);
      else gemm_mma_loop<BN, false>(p, sA, sB, sAcc, full, empty, num_tiles, warp, lane);
    } else {
      gemm_mma_loop<BN, false>(p, sA, sB, sAcc, full, empty, num_tiles, warp, lane);
    }
  } else {
    // ===================== epilogue (1 warpgroup): row r of every tile, all BN columns =====================
    reg_alloc<GEMM_EPI_REGS>();
    const int r = threadIdx.x - GEMM_EPI_THREAD0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
      const int m0 = (tile / n_tiles) * GEMM_BM;
      const int n0 = (tile % n_tiles) * BN;
      named_sync(GEMM_BAR_ACC_FULL, 384);
      if constexpr (EPI == EPI_RESID) epilogue_resid_tile<BN>(p, sAcc, m0, n0, r >> 5, lane);
      else epilogue_tile<BN, EPI>(p, sAcc + r * Cfg::ACC_LD, m0 + r, n0, s_rope);
      if (tile + static_cast<int>(gridDim.x) < num_tiles) named_arrive(GEMM_BAR_ACC_FREE, 384);
    }
  }
}

}  // namespace ovg
