// HBM-bound kernels of the hot path: LayerNorm, token assembly / modality scatter, camera-token injection,
// intermediate snapshots, depth normalisation + im2col, strided-conv im2col, bilinear upsampling.
// All use 16-byte vectorised, coalesced accesses; none reshapes work into GEMMs.
#pragma once
#include "ptx.cuh"

namespace ovg {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// ---------------------------------------------------------------------------------------------------
// LayerNorm over the last dim (reference layers/block.py:50,:67 norm1/norm2; heads/dpt_head.py:66,:227).
// One warp per row; fp32 or bf16 input, bf16 output, optional affine.  Row gather: output row m reads
// input row (m / grp_out) * grp_in + grp_off + (m % grp_out)   (grp_out == 0 -> identity); this drops the 5
// special tokens of every frame for the DPT input (heads/dpt_head.py:219).
enum { LN_IN_F32 = 0, LN_IN_BF16 = 1, LN_IN_F32_AS_BF16 = 2 };
struct LnParams {
  const void* in;
  int in_bf16;      // input type (LN_IN_*): fp32, bf16, or fp32 rounded to bf16 (nearest even) on load -- the values a bf16
                    // snapshot of the same fp32 tensor (inject_snapshot_kernel) would hold
  long long ld_in;
  void* out;
  int out_f32;      // output type: 0 bf16, 1 fp32, 2 IEEE half (saturating)
  long long ld_out;
  int rows, C;
  const float* w;
  const float* b;
  float eps;
  int grp_out, grp_in, grp_off;
};

template <int VPL>
__device__ __forceinline__ void ln_load_row(const LnParams& p, const int row, const int lane, float (&v)[VPL]) {
  long long src = row;
  if (p.grp_out > 0) src = static_cast<long long>(row / p.grp_out) * p.grp_in + p.grp_off + (row % p.grp_out);
  // lane handles chunks of 4 consecutive elements: element index = (i*32 + lane)*4 + e
  if (p.in_bf16 == LN_IN_BF16) {
    const __nv_bfloat16* x = reinterpret_cast<const __nv_bfloat16*>(p.in) + src * p.ld_in;
#pragma unroll
    for (int i = 0; i < VPL / 4; ++i) {
      const uint2 u = *reinterpret_cast<const uint2*>(x + (i * 32 + lane) * 4);
      v[4 * i + 0] = bf16_lo(u.x);
      v[4 * i + 1] = bf16_hi(u.x);
      v[4 * i + 2] = bf16_lo(u.y);
      v[4 * i + 3] = bf16_hi(u.y);
    }
  } else {
    const float* x = reinterpret_cast<const float*>(p.in) + src * p.ld_in;
#pragma unroll
    for (int i = 0; i < VPL / 4; ++i) {
      const float4 f = *reinterpret_cast<const float4*>(x + (i * 32 + lane) * 4);
      v[4 * i + 0] = f.x;
      v[4 * i + 1] = f.y;
      v[4 * i + 2] = f.z;
      v[4 * i + 3] = f.w;
    }
    if (p.in_bf16 == LN_IN_F32_AS_BF16) {
#pragma unroll
      for (int i = 0; i < VPL / 2; ++i) {
        const uint32_t u = pack_bf16(v[2 * i], v[2 * i + 1]);
        v[2 * i] = bf16_lo(u);
        v[2 * i + 1] = bf16_hi(u);
      }
    }
  }
}

// Persistent: the grid is sized to the machine (ovg.cu) and every warp walks rows with a grid stride, loading row i+1
// while it reduces row i, so the HBM stream never drains between "waves" of short-lived blocks.
template <int VPL>  // values per lane = C / 32 (multiple of 4)
__global__ void __launch_bounds__(256, 2) layernorm_kernel(const LnParams p) {
  constexpr bool PF = VPL <= 32;     // two rows of C = 2048 do not fit the register budget of 2 blocks / SM
  const int lane = threadIdx.x & 31;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  int row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (row >= p.rows) return;
  float v[VPL], nx[PF ? VPL : 4];
  if (PF) ln_load_row<VPL>(p, row, lane, v);
  for (; row < p.rows; row += nwarps) {
    const bool more = PF && row + nwarps < p.rows;
    if constexpr (PF) {
      if (more) ln_load_row<VPL>(p, row + nwarps, lane, reinterpret_cast<float (&)[VPL]>(nx));
    } else {
      ln_load_row<VPL>(p, row, lane, v);
    }
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) s += v[i];
    const float mean = warp_sum(s) / p.C;
    float q = 0.f;
#pragma unroll
    for (int i = 0; i < VPL; ++i) {
      const float d = v[i] - mean;
      q += d * d;
    }
    const float rstd = rsqrtf(warp_sum(q) / p.C + p.eps);
#pragma unroll
    for (int i = 0; i < VPL / 4; ++i) {
      const int c = (i * 32 + lane) * 4;
      float o[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) o[e] = (v[4 * i + e] - mean) * rstd;
      if (p.w) {
        const float4 w4 = __ldg(reinterpret_cast<const float4*>(p.w + c));
        const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.b + c));
        o[0] = fmaf(o[0], w4.x, b4.x);
        o[1] = fmaf(o[1], w4.y, b4.y);
        o[2] = fmaf(o[2], w4.z, b4.z);
        o[3] = fmaf(o[3], w4.w, b4.w);
      }
      if (p.out_f32 == 1) {
        *reinterpret_cast<float4*>(reinterpret_cast<float*>(p.out) + static_cast<long long>(row) * p.ld_out + c) =
            make_float4(o[0], o[1], o[2], o[3]);
      } else {
        uint2 u;
        u.x = pack_h(o[0], o[1], p.out_f32 == 2);
        u.y = pack_h(o[2], o[3], p.out_f32 == 2);
        *reinterpret_cast<uint2*>(reinterpret_cast<__nv_bfloat16*>(p.out) + static_cast<long long>(row) * p.ld_out + c) = u;
      }
    }
    if constexpr (PF) {
      if (more) {
#pragma unroll
        for (int i = 0; i < VPL; ++i) v[i] = nx[i];
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// Token assembly (reference omnivggt_aggregator.py:155-156,:211-213 + aggregator.py:343-366).
//   x[k,0]       = camera_token[slot(k)] + inj0[k]              (inj0 = camera_adapters[0](g0), bias on ALL frames)
//   x[k,1..R]    = register_token[slot(k)]
//   x[k,R+1+p]   = patch[k,p] + (has_depth[k] ? 0 : depth_placeholder)   (selected frames get their depth
//                  tokens added by the depth-embedding GEMM epilogue, see ovg_gemm EPI_RESID + row_index)
// slot(k) = 0 for the first view of a scene, 1 otherwise.  One block per token row, float4 per thread.
struct AssembleParams {
  float* x;             // [K, T, C]
  const float* patch;   // [K, P, C]
  const float* cam_tok;  // [2, C]
  const float* reg_tok;  // [2, R, C]
  const float* inj0;     // [K, C]
  const float* placeholder;  // [C]
  const int* has_depth;      // [K]
  int K, S, T, R, C;
  int view_base;             // scene-local index of frame 0 (non-zero only when a scene's views are sharded over ranks)
};

__global__ void assemble_tokens_kernel(const AssembleParams p) {
  const int row = blockIdx.x;
  const int k = row / p.T, t = row % p.T;
  const int slot = ((k % p.S) + p.view_base) == 0 ? 0 : 1;
  const int P = p.T - p.R - 1;
  for (int c = threadIdx.x * 4; c < p.C; c += blockDim.x * 4) {
    float4 o;
    if (t == 0) {
      const float4 a = *reinterpret_cast<const float4*>(p.cam_tok + slot * p.C + c);
      const float4 b = *reinterpret_cast<const float4*>(p.inj0 + static_cast<long long>(k) * p.C + c);
      o = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
    } else if (t <= p.R) {
      o = *reinterpret_cast<const float4*>(p.reg_tok + (static_cast<long long>(slot) * p.R + (t - 1)) * p.C + c);
    } else {
      o = *reinterpret_cast<const float4*>(p.patch + (static_cast<long long>(k) * P + (t - 1 - p.R)) * p.C + c);
      if (!p.has_depth[k]) {
        const float4 d = *reinterpret_cast<const float4*>(p.placeholder + c);
        o.x += d.x; o.y += d.y; o.z += d.z; o.w += d.w;
      }
    }
    *reinterpret_cast<float4*>(p.x + static_cast<long long>(row) * p.C + c) = o;
  }
}

// ---------------------------------------------------------------------------------------------------
// Per-layer camera injection + intermediate snapshot (reference omnivggt_aggregator.py:273-303,:248-251).
//   x[k,0,:] += inj[k,:]                                   (only token 0 of each frame receives a non-zero add)
//   slot[k,t, coff:coff+C] = bf16(x[k,t,:])                (frame half coff=0 / global half coff=C)
//   layer[k,t, coff:coff+C] = x[k,t,:]                     (fp32 export of the layer, as the reference returns it)
//   cam_out[k, coff:coff+C] = x[k,0,:]                     (fp32 camera tokens for the camera head)
struct InjectParams {
  float* x;                 // [K*T, C]
  const float* inj;         // [K, C] or nullptr
  __nv_bfloat16* slot;      // [K*T, 2C] or nullptr
  float* cam_out;           // [K, 2C] or nullptr
  int K, T, C, coff;
  float* layer;             // [K*T, 2C] or nullptr
};

__global__ void inject_snapshot_kernel(const InjectParams p) {
  // with a snapshot slot or layer: one block per token row; without: only the camera-token rows change (one block per frame)
  const int row = (p.slot || p.layer) ? blockIdx.x : blockIdx.x * p.T;
  const int k = row / p.T, t = row % p.T;
  for (int c = threadIdx.x * 4; c < p.C; c += blockDim.x * 4) {
    float4 v = *reinterpret_cast<const float4*>(p.x + static_cast<long long>(row) * p.C + c);
    if (t == 0) {
      if (p.inj) {
        const float4 a = *reinterpret_cast<const float4*>(p.inj + static_cast<long long>(k) * p.C + c);
        v.x += a.x; v.y += a.y; v.z += a.z; v.w += a.w;
        *reinterpret_cast<float4*>(p.x + static_cast<long long>(row) * p.C + c) = v;
      }
      if (p.cam_out) *reinterpret_cast<float4*>(p.cam_out + static_cast<long long>(k) * 2 * p.C + p.coff + c) = v;
    }
    if (p.slot) {
      uint2 u;
      u.x = pack_bf16(v.x, v.y);
      u.y = pack_bf16(v.z, v.w);
      *reinterpret_cast<uint2*>(p.slot + static_cast<long long>(row) * 2 * p.C + p.coff + c) = u;
    }
    if (p.layer) *reinterpret_cast<float4*>(p.layer + static_cast<long long>(row) * 2 * p.C + p.coff + c) = v;
  }
}

// ---------------------------------------------------------------------------------------------------
// Depth modality (reference omnivggt_aggregator.py:107-128,:189-199): per-scene masked mean over the
// selected views, then im2col of [depth/(mean+eps)*mask, mask] into rows of 2*14*14 for the 14x14/s14
// patch-embedding GEMM.  Two deterministic stages (no float atomics).
struct DepthParams {
  const float* depth;  // [B, S, H, W]
  const float* mask;   // [B, S, H, W]
  const int* idx;      // [Sd] selected views
  double* partial;     // [B, NCHUNK, 2] (sum, count), then [B] scale factors as float at partial + B * NCHUNK * 2
  __nv_bfloat16* cols;  // [B*Sd*hp*wp, ldc]
  int ldc;
  int B, S, Sd, H, W, patch;
};
constexpr int DEPTH_NCHUNK = 1024;

// Stage 1: 1024 blocks per scene, each sums a contiguous run of float2 pairs of the selected views (H * W is even: both are
// multiples of the even patch size).  fp32 partial sums over <= 64 values per thread, combined in double.
__global__ void __launch_bounds__(256) depth_stats_kernel(const DepthParams p) {
  const int b = blockIdx.y, ch = blockIdx.x;
  const long long per2 = static_cast<long long>(p.H) * p.W / 2;
  const long long total2 = per2 * p.Sd;
  const long long span = (total2 + DEPTH_NCHUNK - 1) / DEPTH_NCHUNK;
  const long long lo = ch * span, hi = min(lo + span, total2);
  double s = 0.0, cnt = 0.0;
  float fs = 0.f, fc = 0.f;
  int run = 0;
  for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    const int j = static_cast<int>(i / per2);
    const long long off = (static_cast<long long>(b) * p.S + p.idx[j]) * per2 + (i - j * per2);
    const float2 m = reinterpret_cast<const float2*>(p.mask)[off];
    const float2 d = reinterpret_cast<const float2*>(p.depth)[off];
    if (m.x > 0.f) { fs += d.x; fc += 1.f; }
    if (m.y > 0.f) { fs += d.y; fc += 1.f; }
    if (++run == 32) {
      s += fs; cnt += fc; fs = 0.f; fc = 0.f; run = 0;
    }
  }
  s += fs;
  cnt += fc;
  __shared__ double sh[2][256];
  sh[0][threadIdx.x] = s;
  sh[1][threadIdx.x] = cnt;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      sh[0][threadIdx.x] += sh[0][threadIdx.x + o];
      sh[1][threadIdx.x] += sh[1][threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    p.partial[(static_cast<long long>(b) * DEPTH_NCHUNK + ch) * 2 + 0] = sh[0][0];
    p.partial[(static_cast<long long>(b) * DEPTH_NCHUNK + ch) * 2 + 1] = sh[1][0];
  }
}

// Stage 2: one block per scene folds the partials in a fixed order -> scale = 1 / (mean + 1e-8), or 0 without a valid pixel.
__global__ void __launch_bounds__(256) depth_scale_kernel(const DepthParams p) {
  const int b = blockIdx.x;
  __shared__ double sh[2][256];
  double s = 0.0, c = 0.0;
  for (int i = threadIdx.x; i < DEPTH_NCHUNK; i += 256) {
    s += p.partial[(static_cast<long long>(b) * DEPTH_NCHUNK + i) * 2 + 0];
    c += p.partial[(static_cast<long long>(b) * DEPTH_NCHUNK + i) * 2 + 1];
  }
  sh[0][threadIdx.x] = s;
  sh[1][threadIdx.x] = c;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      sh[0][threadIdx.x] += sh[0][threadIdx.x + o];
      sh[1][threadIdx.x] += sh[1][threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    float* scale = reinterpret_cast<float*>(p.partial + static_cast<long long>(p.B) * DEPTH_NCHUNK * 2);
    scale[b] = sh[1][0] > 0.0 ? 1.0f / (static_cast<float>(sh[0][0] / sh[1][0]) + 1e-8f) : 0.0f;   // no valid pixel -> zeros (:121-122)
  }
}

// Stage 3: one block per (scene, selected view, patch row): the 14 image rows are read as coalesced float2 runs, every pair
// lands in one patch (the patch size is even) and is stored as one bf16x2.
template <int PATCH>      // compile-time patch size (0: runtime p.patch): the index arithmetic is half of this kernel's instructions
__global__ void __launch_bounds__(256) depth_im2col_kernel(const DepthParams pin) {
  DepthParams p = pin;
  if (PATCH > 0) p.patch = PATCH;
  const int hp = p.H / p.patch, wp = p.W / p.patch;
  const int py = blockIdx.x % hp, j = (blockIdx.x / hp) % p.Sd, b = blockIdx.x / (hp * p.Sd);
  const float scale = reinterpret_cast<const float*>(p.partial + static_cast<long long>(p.B) * DEPTH_NCHUNK * 2)[b];
  const int w2 = p.W / 2, pp = p.patch * p.patch;
  const long long img = ((static_cast<long long>(b) * p.S + p.idx[j]) * p.H + static_cast<long long>(py) * p.patch) * p.W;
  const long long row0 = ((static_cast<long long>(b) * p.Sd + j) * hp + py) * wp;
  for (int e = threadIdx.x; e < p.patch * w2; e += blockDim.x) {
    const int ky = e / w2, x = (e - ky * w2) * 2;
    const int px = x / p.patch, kx = x - px * p.patch;
    const long long off = img + static_cast<long long>(ky) * p.W + x;
    const float2 m = *reinterpret_cast<const float2*>(p.mask + off);
    const float2 d = *reinterpret_cast<const float2*>(p.depth + off);
    __nv_bfloat16* dst = p.cols + (row0 + px) * p.ldc + ky * p.patch + kx;
    *reinterpret_cast<uint32_t*>(dst) = pack_bf16(d.x * scale * m.x, d.y * scale * m.y);
    *reinterpret_cast<uint32_t*>(dst + pp) = pack_bf16(m.x, m.y);
  }
}

// ---------------------------------------------------------------------------------------------------
// RGB patch im2col for the DINOv2 patch-embedding GEMM (reference layers/patch_embed.py:65-77) with the ImageNet
// normalisation of models/omnivggt_aggregator.py:143 fused.  One block per (frame, patch row): 3 x 14 image rows as coalesced
// float2 runs -> bf16x2 stores into cols (c, ky, kx); columns [3 * patch^2, ldc) are zero padding.
struct ImageColParams {
  const float* img;   // [K, 3, H, W]
  __nv_bfloat16* cols;
  int ldc, K, H, W, patch;
  float mean[3], istd[3];
};

template <int PATCH>
__global__ void __launch_bounds__(256) image_im2col_kernel(const ImageColParams pin) {
  ImageColParams p = pin;
  if (PATCH > 0) p.patch = PATCH;
  const int hp = p.H / p.patch, wp = p.W / p.patch;
  const int py = blockIdx.x % hp, k = blockIdx.x / hp;
  const int w2 = p.W / 2, pp = p.patch * p.patch;
  const long long row0 = (static_cast<long long>(k) * hp + py) * wp;
  const int per_c = p.patch * w2;
  for (int e = threadIdx.x; e < 3 * per_c; e += blockDim.x) {
    const int c = e / per_c, r = e - c * per_c;
    const int ky = r / w2, x = (r - ky * w2) * 2;
    const int px = x / p.patch, kx = x - px * p.patch;
    const float2 v = *reinterpret_cast<const float2*>(
        p.img + ((static_cast<long long>(k) * 3 + c) * p.H + (py * p.patch + ky)) * p.W + x);
    *reinterpret_cast<uint32_t*>(p.cols + (row0 + px) * p.ldc + c * pp + ky * p.patch + kx) =
        pack_bf16((v.x - p.mean[c]) * p.istd[c], (v.y - p.mean[c]) * p.istd[c]);
  }
  const int padw = p.ldc - 3 * pp;      // even: ldc % 8 == 0 and 3 * patch^2 is even
  for (int e = threadIdx.x; e < wp * (padw / 2); e += blockDim.x) {
    const int px = e / (padw / 2), q = e - px * (padw / 2);
    *reinterpret_cast<uint32_t*>(p.cols + (row0 + px) * p.ldc + 3 * pp + 2 * q) = 0u;
  }
}

// ---------------------------------------------------------------------------------------------------
// im2col for the stride-2 3x3 conv of DPT level 4 (reference heads/dpt_head.py:93-95): dense NHWC
// [F,h,w,C] -> rows (f,oy,ox) x cols (tap, c).  One block per (output pixel, tap); uint4 copies.
struct Im2colParams {
  const __nv_bfloat16* src;  // [F, h, w, C]
  __nv_bfloat16* dst;        // [F*oh*ow, 9*C]
  int F, h, w, C, oh, ow;
};

__global__ void im2col3x3s2_kernel(const Im2colParams p) {
  const int tap = blockIdx.y;
  const int pix = blockIdx.x;
  const int ox = pix % p.ow, oy = (pix / p.ow) % p.oh, f = pix / (p.ow * p.oh);
  const int iy = 2 * oy + tap / 3 - 1, ix = 2 * ox + tap % 3 - 1;
  const bool ok = iy >= 0 && iy < p.h && ix >= 0 && ix < p.w;
  const uint4* s = reinterpret_cast<const uint4*>(p.src + ((static_cast<long long>(f) * p.h + iy) * p.w + ix) * p.C);
  uint4* d = reinterpret_cast<uint4*>(p.dst + (static_cast<long long>(pix) * 9 + tap) * p.C);
  for (int c = threadIdx.x; c < p.C / 8; c += blockDim.x) d[c] = ok ? s[c] : make_uint4(0, 0, 0, 0);
}

// ---------------------------------------------------------------------------------------------------
// Bilinear upsampling, align_corners=True (reference heads/dpt_head.py:466,:472-497, F.interpolate), on
// zero-bordered NHWC bf16 maps: src [F,h+2,w+2,C] -> dst [F,H+2,W+2,C].  Optional additive UV position embedding
// (heads/dpt_head.py:249-250): the sin/cos embedding of heads/utils.py:11-108 is separable -- channels [0,C/2) depend on x
// only, [C/2,C) on y only -- so it is passed as two small tables tx [W, C/2], ty [H, C/2] (x0.1 folded in) instead of an
// [H*W, C] fp32 map that would have to be streamed from HBM for every frame.  Border pixels are written as 0.
// Grid (x-chunks, H+2, F): no integer divisions in the index math; each thread moves 8 channels (16 B).
struct UpsampleParams {
  const __nv_bfloat16* src;
  __nv_bfloat16* dst;
  const float* tx;
  const float* ty;
  int F, h, w, H, W, C;
  float sy, sx;
  int f16;          // maps are IEEE half instead of bf16
};

__global__ void __launch_bounds__(256) upsample_bilinear_kernel(const UpsampleParams p) {
  const int vec = p.C >> 3;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  const int X = t / vec;
  const int cv = t - X * vec;
  if (X >= p.W + 2) return;
  const int Y = blockIdx.y, f = blockIdx.z;
  uint4 out = make_uint4(0, 0, 0, 0);
  if (X >= 1 && X <= p.W && Y >= 1 && Y <= p.H) {
    const int oy = Y - 1, ox = X - 1;
    const float fy = p.sy * oy, fx = p.sx * ox;
    const int y0 = static_cast<int>(fy), x0 = static_cast<int>(fx);
    const int y1 = y0 + (y0 < p.h - 1 ? 1 : 0), x1 = x0 + (x0 < p.w - 1 ? 1 : 0);
    const float wy1 = fy - y0, wx1 = fx - x0;
    const float wy0 = 1.f - wy1, wx0 = 1.f - wx1;
    const __nv_bfloat16* base = p.src + static_cast<size_t>(f) * (p.h + 2) * (p.w + 2) * p.C;
    const int ws = p.w + 2;
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(base + static_cast<size_t>((y0 + 1) * ws + (x0 + 1)) * p.C) + cv);
    const uint4 b = __ldg(reinterpret_cast<const uint4*>(base + static_cast<size_t>((y0 + 1) * ws + (x1 + 1)) * p.C) + cv);
    const uint4 c = __ldg(reinterpret_cast<const uint4*>(base + static_cast<size_t>((y1 + 1) * ws + (x0 + 1)) * p.C) + cv);
    const uint4 d = __ldg(reinterpret_cast<const uint4*>(base + static_cast<size_t>((y1 + 1) * ws + (x1 + 1)) * p.C) + cv);
    const uint32_t* ap = &a.x; const uint32_t* bp = &b.x; const uint32_t* cp = &c.x; const uint32_t* dp = &d.x;
    float r[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float2 va = unpack_h(ap[i], p.f16), vb = unpack_h(bp[i], p.f16), vc = unpack_h(cp[i], p.f16), vd = unpack_h(dp[i], p.f16);
      r[2 * i] = wy0 * (wx0 * va.x + wx1 * vb.x) + wy1 * (wx0 * vc.x + wx1 * vd.x);
      r[2 * i + 1] = wy0 * (wx0 * va.y + wx1 * vb.y) + wy1 * (wx0 * vc.y + wx1 * vd.y);
    }
    if (p.tx) {
      const int half = p.C >> 1;
      const int c0 = cv * 8;
      const float* tp = c0 < half ? p.tx + static_cast<size_t>(ox) * half + c0 : p.ty + static_cast<size_t>(oy) * half + (c0 - half);
      const float4 t0 = __ldg(reinterpret_cast<const float4*>(tp)), t1 = __ldg(reinterpret_cast<const float4*>(tp) + 1);
      r[0] += t0.x; r[1] += t0.y; r[2] += t0.z; r[3] += t0.w;
      r[4] += t1.x; r[5] += t1.y; r[6] += t1.z; r[7] += t1.w;
    }
    out.x = pack_h(r[0], r[1], p.f16);
    out.y = pack_h(r[2], r[3], p.f16);
    out.z = pack_h(r[4], r[5], p.f16);
    out.w = pack_h(r[6], r[7], p.f16);
  }
  *(reinterpret_cast<uint4*>(p.dst + (static_cast<size_t>(f) * (p.H + 2) * (p.W + 2) + static_cast<size_t>(Y) * (p.W + 2) + X) * p.C) + cv) = out;
}

// Row-wise two-pass variant (default): one block per (output row, frame, 32-channel group).  Pass 1 blends the two
// source rows vertically into shared memory once (fp32), pass 2 blends horizontally out of shared memory.  The direct
// kernel above gathers four source texels per output and spends most of its issue slots unpacking bf16 (ncu: issue 76 %,
// ALU pipe 62 %, 2.0 TB/s); here every source texel is loaded and unpacked once per output row.
__global__ void __launch_bounds__(256) upsample_rows_kernel(const UpsampleParams p) {
  extern __shared__ float srow[];                       // [w][32]
  const int Y = blockIdx.x, f = blockIdx.y, cg = blockIdx.z;
  const int Wp = p.W + 2;
  __nv_bfloat16* drow = p.dst + (static_cast<size_t>(f) * (p.H + 2) + Y) * Wp * p.C + cg * 32;
  if (Y == 0 || Y == p.H + 1) {                         // zero border row
    for (int i = threadIdx.x; i < Wp * 4; i += blockDim.x)
      *reinterpret_cast<uint4*>(drow + static_cast<size_t>(i >> 2) * p.C + (i & 3) * 8) = make_uint4(0, 0, 0, 0);
    return;
  }
  const int oy = Y - 1;
  const float fy = p.sy * oy;
  const int y0 = static_cast<int>(fy);
  const int y1 = y0 + (y0 < p.h - 1 ? 1 : 0);
  const float wy1 = fy - y0, wy0 = 1.f - wy1;
  const int ws = p.w + 2;
  const __nv_bfloat16* fbase = p.src + static_cast<size_t>(f) * (p.h + 2) * ws * p.C + cg * 32;
  const __nv_bfloat16* s0 = fbase + (static_cast<size_t>(y0 + 1) * ws + 1) * p.C;
  const __nv_bfloat16* s1 = fbase + (static_cast<size_t>(y1 + 1) * ws + 1) * p.C;
  for (int i = threadIdx.x; i < p.w * 4; i += blockDim.x) {
    const int x = i >> 2, v = i & 3;
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(s0 + static_cast<size_t>(x) * p.C) + v);
    const uint4 b = __ldg(reinterpret_cast<const uint4*>(s1 + static_cast<size_t>(x) * p.C) + v);
    const uint32_t* ap = &a.x;
    const uint32_t* bp = &b.x;
    float r[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 va = unpack_h(ap[k], p.f16), vb = unpack_h(bp[k], p.f16);
      r[2 * k] = wy0 * va.x + wy1 * vb.x;
      r[2 * k + 1] = wy0 * va.y + wy1 * vb.y;
    }
    float4* d = reinterpret_cast<float4*>(srow + x * 32 + v * 8);
    d[0] = make_float4(r[0], r[1], r[2], r[3]);
    d[1] = make_float4(r[4], r[5], r[6], r[7]);
  }
  __syncthreads();
  const int half = p.C >> 1;
  for (int i = threadIdx.x; i < Wp * 4; i += blockDim.x) {
    const int X = i >> 2, v = i & 3;
    uint4 out = make_uint4(0, 0, 0, 0);
    if (X >= 1 && X <= p.W) {
      const int ox = X - 1;
      const float fx = p.sx * ox;
      const int x0 = static_cast<int>(fx);
      const int x1 = x0 + (x0 < p.w - 1 ? 1 : 0);
      const float wx1 = fx - x0, wx0 = 1.f - wx1;
      const float4* a = reinterpret_cast<const float4*>(srow + x0 * 32 + v * 8);
      const float4* b = reinterpret_cast<const float4*>(srow + x1 * 32 + v * 8);
      const float4 a0 = a[0], a1 = a[1], b0 = b[0], b1 = b[1];
      float r[8] = {wx0 * a0.x + wx1 * b0.x, wx0 * a0.y + wx1 * b0.y, wx0 * a0.z + wx1 * b0.z, wx0 * a0.w + wx1 * b0.w,
                    wx0 * a1.x + wx1 * b1.x, wx0 * a1.y + wx1 * b1.y, wx0 * a1.z + wx1 * b1.z, wx0 * a1.w + wx1 * b1.w};
      if (p.tx) {
        const int c0 = cg * 32 + v * 8;
        const float* tp = c0 < half ? p.tx + static_cast<size_t>(ox) * half + c0 : p.ty + static_cast<size_t>(oy) * half + (c0 - half);
        const float4 t0 = __ldg(reinterpret_cast<const float4*>(tp)), t1 = __ldg(reinterpret_cast<const float4*>(tp) + 1);
        r[0] += t0.x; r[1] += t0.y; r[2] += t0.z; r[3] += t0.w;
        r[4] += t1.x; r[5] += t1.y; r[6] += t1.z; r[7] += t1.w;
      }
      out.x = pack_h(r[0], r[1], p.f16);
      out.y = pack_h(r[2], r[3], p.f16);
      out.z = pack_h(r[4], r[5], p.f16);
      out.w = pack_h(r[6], r[7], p.f16);
    }
    *reinterpret_cast<uint4*>(drow + static_cast<size_t>(X) * p.C + v * 8) = out;
  }
}

// ---------------------------------------------------------------------------------------------------
// Cross-GPU barrier on peer-mapped flags (context-parallel global attention): the K / V rows a rank stored into its peers'
// buffers (QKV epilogue of the kernels before this one on the stream) become visible before any peer's attention reads them.
// Rows of this rank -> the same row window of every peer's buffer (camera tokens of a sharded scene; a few KB).
struct PeerRowsParams {
  const float* src;     // [rows, width]
  float* dst[8];        // per rank: [rows_total, width], peer mapped
  int world, rows, width;
  long long row_off;
};
__global__ void peer_rows_kernel(const PeerRowsParams p) {
  const long long n4 = static_cast<long long>(p.rows) * p.width / 4;
  float4* d = reinterpret_cast<float4*>(p.dst[blockIdx.y] + p.row_off * p.width);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x)
    d[i] = reinterpret_cast<const float4*>(p.src)[i];
}

struct PeerBarrierParams {
  int* flags[8];     // flags[r]: int[world] in rank r's memory (peer mapped)
  int* epoch;        // this rank's private barrier counter (device memory): every barrier uses the next value, so a captured
                     // CUDA graph can be replayed (no epoch baked into the launch)
  int rank, world;
};
__global__ void peer_barrier_kernel(const PeerBarrierParams p) {
  const int t = threadIdx.x;
  __shared__ int s_epoch;
  if (t == 0) {
    s_epoch = *p.epoch + 1;
    *p.epoch = s_epoch;
  }
  __syncthreads();
  const int epoch = s_epoch;
  if (t < p.world) {
    __threadfence_system();                                   // peer stores of earlier kernels are complete at kernel end; order the flag after them
    volatile int* remote = p.flags[t] + p.rank;
    *remote = epoch;
    __threadfence_system();
    volatile int* mine = p.flags[p.rank] + t;
    long long spins = 0;
    while (*mine < epoch) {
      if (++spins > 2000000000LL) __trap();                   // a rank that never arrives must not hang the box silently
    }
    __threadfence_system();
  }
}

}  // namespace ovg
