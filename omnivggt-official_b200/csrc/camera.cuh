// Small kernels of the camera head (reference heads/camera_head.py:83-154): M = B*S rows (8 .. a few dozen), so everything
// except the weight-streaming GEMMs (which run on the wgmma GEMM of gemm.cuh) is a one-warp-per-row kernel in fp32.
#pragma once
#include "elem.cuh"

namespace ovg {

// e = SiLU(W_e p + b_e) for p = the previous pose encoding (or the learned empty pose token): [K, 9] -> bf16 [K, D]
// (camera_head.py:124-129: embed_pose, then the SiLU in front of poseLN_modulation's Linear).
struct PoseEmbedParams {
  const float* pose;     // [K, 9] or nullptr (first iteration: empty_pose broadcast)
  const float* empty;    // [9]
  const float* w;        // [D, 9]
  const float* b;        // [D]
  __nv_bfloat16* out;    // [K, D]
  int K, D;
};
__global__ void pose_embed_silu_kernel(const PoseEmbedParams p) {
  const long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
  if (i >= static_cast<long long>(p.K) * p.D) return;
  const int k = static_cast<int>(i / p.D), c = static_cast<int>(i % p.D);
  const float* x = p.pose ? p.pose + k * 9 : p.empty;
  float acc = p.b[c];
#pragma unroll
  for (int j = 0; j < 9; ++j) acc += p.w[c * 9 + j] * x[j];
  p.out[i] = __float2bfloat16(acc / (1.0f + __expf(-acc)));
}

// h = gate * (LN_1e-6(tok) * (1 + scale) + shift) + tok       (camera_head.py:131-136,:157-162; adaln_norm has no affine)
struct AdaLnParams {
  const float* tok;              // [K, D] fp32 (token_norm output)
  const __nv_bfloat16* mod;      // [K, 3D] = [shift | scale | gate]
  float* h;                      // [K, D]
  int K, D;
};
__global__ void __launch_bounds__(128) adaln_modulate_kernel(const AdaLnParams p) {
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= p.K) return;
  const float* t = p.tok + static_cast<long long>(row) * p.D;
  float s = 0.f;
  for (int c = lane; c < p.D; c += 32) s += t[c];
  const float mean = warp_sum(s) / p.D;
  float q = 0.f;
  for (int c = lane; c < p.D; c += 32) {
    const float d = t[c] - mean;
    q += d * d;
  }
  const float rstd = rsqrtf(warp_sum(q) / p.D + 1e-6f);
  const __nv_bfloat16* m = p.mod + static_cast<long long>(row) * 3 * p.D;
  for (int c = lane; c < p.D; c += 32) {
    const float xh = (t[c] - mean) * rstd;
    const float shift = __bfloat162float(m[c]), scale = __bfloat162float(m[p.D + c]), gate = __bfloat162float(m[2 * p.D + c]);
    p.h[static_cast<long long>(row) * p.D + c] = gate * (xh * (1.0f + scale) + shift) + t[c];
  }
}

// Attention across the S camera tokens of a scene: one warp per (row, head), online softmax in fp32, head_dim = 32 * DPL.
// qkv: bf16 [K, 3 * D] as written by the plain QKV GEMM = [q | k | v][heads][hd]  (layers/attention.py:52-66, no RoPE / q-k norm).
struct SmallAttnParams {
  const __nv_bfloat16* qkv;
  __nv_bfloat16* out;     // [K, D]
  int K, S, heads, hd;
  float scale;
};
template <int DPL>
__global__ void __launch_bounds__(128) small_attention_kernel(const SmallAttnParams p) {
  const int w = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= p.K * p.heads) return;
  const int row = w / p.heads, head = w % p.heads;
  const int D = p.heads * p.hd;
  const int scene0 = (row / p.S) * p.S;
  float q[DPL], acc[DPL];
#pragma unroll
  for (int d = 0; d < DPL; ++d) {
    q[d] = __bfloat162float(p.qkv[static_cast<long long>(row) * 3 * D + head * p.hd + lane * DPL + d]) * p.scale;
    acc[d] = 0.f;
  }
  float m = -INFINITY, l = 0.f;
  for (int j = 0; j < p.S; ++j) {
    const __nv_bfloat16* kv = p.qkv + static_cast<long long>(scene0 + j) * 3 * D + head * p.hd + lane * DPL;
    float s = 0.f;
#pragma unroll
    for (int d = 0; d < DPL; ++d) s += q[d] * __bfloat162float(kv[D + d]);
    s = warp_sum(s);
    const float mn = fmaxf(m, s);
    const float a = __expf(m - mn), e = __expf(s - mn);
    l = l * a + e;
#pragma unroll
    for (int d = 0; d < DPL; ++d) acc[d] = acc[d] * a + e * __bfloat162float(kv[2 * D + d]);
    m = mn;
  }
  const float inv = 1.0f / l;
#pragma unroll
  for (int d = 0; d < DPL; ++d)
    p.out[static_cast<long long>(row) * D + head * p.hd + lane * DPL + d] = __float2bfloat16(acc[d] * inv);
}

// delta = W2 g + b2 (hidden -> 9), pose += delta (first iteration: pose = delta), activated = [t, quat linear; fov relu]
// (camera_head.py:139-152, layers/mlp.py:38, heads/head_act.py:12-35).
struct PoseOutParams {
  const __nv_bfloat16* g;   // [K, hidden] = GELU(fc1(...))
  const float* w2;          // [9, hidden]
  const float* b2;          // [9]
  float* pose;              // [K, 9] running (un-activated) prediction, updated in place
  float* out;               // [K, 9] activated prediction of this iteration
  int K, hidden, first;
};
__global__ void __launch_bounds__(128) pose_out_kernel(const PoseOutParams p) {
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= p.K) return;
  const __nv_bfloat16* g = p.g + static_cast<long long>(row) * p.hidden;
  float acc[9];
#pragma unroll
  for (int j = 0; j < 9; ++j) acc[j] = 0.f;
  for (int c = lane; c < p.hidden; c += 32) {
    const float v = __bfloat162float(g[c]);
#pragma unroll
    for (int j = 0; j < 9; ++j) acc[j] += p.w2[j * p.hidden + c] * v;
  }
#pragma unroll
  for (int j = 0; j < 9; ++j) acc[j] = warp_sum(acc[j]);
  if (lane < 9) {
    float v = 0.f;
#pragma unroll
    for (int j = 0; j < 9; ++j)
      if (j == lane) v = acc[j];
    v += p.b2[lane];
    if (!p.first) v += p.pose[row * 9 + lane];
    p.pose[row * 9 + lane] = v;
    p.out[row * 9 + lane] = lane >= 7 ? fmaxf(v, 0.f) : v;
  }
}

}  // namespace ovg
