// On-device post-processing of the predictions (SURVEY.md section 8f rank 3): the step right after the hot path, which the
// reference does on the host with numpy (inference.py:360-365,:132-133; visual_util.py:42-73).
//   pose_decode_kernel        pose_enc -> [R|t] world->camera, pinhole K, camera->world        (utils/pose_enc.py:65-130,
//                                                                    utils/rotation.py:14-44, utils/geometry.py:269-318)
//   unproject_kernel          depth + cameras -> world points                                  (utils/geometry.py:151-264)
//   percentile select + mask  conf >= percentile(conf, p) && conf > 0.1                        (inference.py:132-133)
//   cloud_* kernels           background filters, ordered compaction, centre, scene scale      (visual_util.py:190-236,
//                                                                    inference.py:96-151)
// All HBM-bound: one coalesced pass per kernel, 16-byte accesses where the layout allows; the percentile is an exact
// order statistic by 4 x 8-bit radix-select passes over the fp32 bit patterns (integer histograms: deterministic).
#pragma once
#include "compact.cuh"
#include "ptx.cuh"

namespace ovg {

// ---------------------------------------------------------------------------------------------------
struct PoseDecodeParams {
  const float* pose_enc;  // [K, 9] = [t(3), quat xyzw(4), fov_h, fov_w]
  float* extrinsic;       // [K, 3, 4] world -> camera
  float* intrinsic;       // [K, 3, 3]
  float* cam2world;       // [K, 3, 4] inverse of extrinsic (closed form: R^T, -R^T t)
  int K;
  float H, W;
};

__global__ void pose_decode_kernel(const PoseDecodeParams p) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= p.K) return;
  const float* e = p.pose_enc + k * 9;
  const float tx = e[0], ty = e[1], tz = e[2];
  const float i = e[3], j = e[4], kk = e[5], r = e[6];
  const float two_s = 2.0f / (i * i + j * j + kk * kk + r * r);       // utils/rotation.py:29 (quaternion need not be unit)
  float R[9];
  R[0] = 1.0f - two_s * (j * j + kk * kk);
  R[1] = two_s * (i * j - kk * r);
  R[2] = two_s * (i * kk + j * r);
  R[3] = two_s * (i * j + kk * r);
  R[4] = 1.0f - two_s * (i * i + kk * kk);
  R[5] = two_s * (j * kk - i * r);
  R[6] = two_s * (i * kk - j * r);
  R[7] = two_s * (j * kk + i * r);
  R[8] = 1.0f - two_s * (i * i + j * j);
  float* x = p.extrinsic + k * 12;
  const float t[3] = {tx, ty, tz};
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    x[a * 4 + 0] = R[a * 3 + 0];
    x[a * 4 + 1] = R[a * 3 + 1];
    x[a * 4 + 2] = R[a * 3 + 2];
    x[a * 4 + 3] = t[a];
  }
  if (p.intrinsic) {
    float* m = p.intrinsic + k * 9;
    const float fy = (p.H * 0.5f) / tanf(e[7] * 0.5f);               // utils/pose_enc.py:118-119
    const float fx = (p.W * 0.5f) / tanf(e[8] * 0.5f);
    m[0] = fx;  m[1] = 0.f; m[2] = p.W * 0.5f;
    m[3] = 0.f; m[4] = fy;  m[5] = p.H * 0.5f;
    m[6] = 0.f; m[7] = 0.f; m[8] = 1.0f;
  }
  if (p.cam2world) {
    float* c = p.cam2world + k * 12;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      c[a * 4 + 0] = R[0 * 3 + a];
      c[a * 4 + 1] = R[1 * 3 + a];
      c[a * 4 + 2] = R[2 * 3 + a];
      c[a * 4 + 3] = -(R[0 * 3 + a] * tx + R[1 * 3 + a] * ty + R[2 * 3 + a] * tz);
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// world[k, v, u, :] = R_c2w ((u - cu) d / fu, (v - cv) d / fv, d) + t_c2w.  4 pixels per thread: one float4 depth load,
// three float4 stores (48 contiguous bytes).  4 B read + 12 B written per pixel.
struct UnprojectParams {
  const float* depth;      // [K, H, W]
  const float* intrinsic;  // [K, 3, 3]
  const float* cam2world;  // [K, 3, 4]
  float* world;            // [K, H, W, 3]
  int K, H, W;             // W % 4 == 0 is not required (scalar tail)
};

__global__ void __launch_bounds__(256) unproject_kernel(const UnprojectParams p) {
  const int k = blockIdx.y;
  const long long hw = static_cast<long long>(p.H) * p.W;
  const float* m = p.intrinsic + k * 9;
  const float* c = p.cam2world + k * 12;
  const float ifu = 1.0f / m[0], ifv = 1.0f / m[4], cu = m[2], cv = m[5];
  const float r00 = c[0], r01 = c[1], r02 = c[2], t0 = c[3];
  const float r10 = c[4], r11 = c[5], r12 = c[6], t1 = c[7];
  const float r20 = c[8], r21 = c[9], r22 = c[10], t2 = c[11];
  const float* d = p.depth + k * hw;
  float* w = p.world + k * hw * 3;
  const bool vec = (hw % 4 == 0) && (p.W % 4 == 0);
  const long long nq = (hw + 3) / 4;
  for (long long q = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; q < nq;
       q += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long i0 = q * 4;
    float dv[4];
    if (vec) {
      const float4 f = *reinterpret_cast<const float4*>(d + i0);
      dv[0] = f.x; dv[1] = f.y; dv[2] = f.z; dv[3] = f.w;
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) dv[e] = i0 + e < hw ? d[i0 + e] : 0.f;
    }
    float o[12];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const long long i = i0 + e;
      const int v = static_cast<int>(i / p.W), u = static_cast<int>(i - static_cast<long long>(v) * p.W);
      // the reference divides by the focal length (x = (u - cu) * d / fu, numpy fp32/fp64 mix); 1 / fu is exact to 1 ulp
      const float xc = (static_cast<float>(u) - cu) * dv[e] * ifu;
      const float yc = (static_cast<float>(v) - cv) * dv[e] * ifv;
      const float zc = dv[e];
      o[3 * e + 0] = r00 * xc + r01 * yc + r02 * zc + t0;
      o[3 * e + 1] = r10 * xc + r11 * yc + r12 * zc + t1;
      o[3 * e + 2] = r20 * xc + r21 * yc + r22 * zc + t2;
    }
    if (vec) {
      float4* dst = reinterpret_cast<float4*>(w + i0 * 3);
      dst[0] = make_float4(o[0], o[1], o[2], o[3]);
      dst[1] = make_float4(o[4], o[5], o[6], o[7]);
      dst[2] = make_float4(o[8], o[9], o[10], o[11]);
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e)
        if (i0 + e < hw) {
          w[(i0 + e) * 3 + 0] = o[3 * e + 0];
          w[(i0 + e) * 3 + 1] = o[3 * e + 1];
          w[(i0 + e) * 3 + 2] = o[3 * e + 2];
        }
    }
  }
}

// ---------------------------------------------------------------------------------------------------
// Exact order statistics of N fp32 values by radix select on the monotone key (sign-flipped bit pattern), 8 bits per pass,
// most significant first.  state[0..1] = the two target ranks (0-based, ascending), state[2..3] = their key prefixes,
// state[4..5] = ranks within the current prefix bucket.  hist: [2][256] counters, zeroed by the decide step.
__device__ __forceinline__ uint32_t f32_key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_f32(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

struct SelectParams {
  const float* v;
  long long n;
  unsigned long long* state;   // [0..1] target ranks, [2..3] prefixes (as u64), [4..5] residual ranks
  unsigned int* hist;          // [2][256]
  int pass;                    // 0..3
  float* out;                  // [2] selected values (written after the last pass), [2] = interpolated threshold
  float frac;                  // linear interpolation weight between the two order statistics (numpy 'linear')
};

// Ranks, empty prefixes, zeroed histograms and kept-counter: one tiny launch instead of host-side copies (graph-capturable).
__global__ void select_init_kernel(unsigned long long* state, unsigned int* hist, unsigned long long r0, unsigned long long r1,
                                   unsigned long long* count) {
  if (threadIdx.x == 0) {
    state[0] = r0; state[1] = r1; state[2] = 0; state[3] = 0; state[4] = r0; state[5] = r1;
    if (count) *count = 0;
  }
  for (int i = threadIdx.x; i < 512; i += blockDim.x) hist[i] = 0;
}

__global__ void __launch_bounds__(256) select_hist_kernel(const SelectParams p) {
  __shared__ unsigned int sh[2][256];
  sh[0][threadIdx.x] = 0;
  sh[1][threadIdx.x] = 0;
  __syncthreads();
  const int shift = 24 - 8 * p.pass;
  const uint32_t mask_hi = p.pass == 0 ? 0u : (0xffffffffu << (shift + 8));
  const uint32_t pre0 = static_cast<uint32_t>(p.state[2]), pre1 = static_cast<uint32_t>(p.state[3]);
  const bool same = pre0 == pre1;
  const long long n4 = p.n / 4;
  const float4* v4 = reinterpret_cast<const float4*>(p.v);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 f = v4[i];
    const float e[4] = {f.x, f.y, f.z, f.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t key = f32_key(e[j]);
      if ((key & mask_hi) == pre0) atomicAdd(&sh[0][(key >> shift) & 255], 1u);
      if (!same && (key & mask_hi) == pre1) atomicAdd(&sh[1][(key >> shift) & 255], 1u);
    }
  }
  if (blockIdx.x == 0) {
    for (long long i = n4 * 4 + threadIdx.x; i < p.n; i += blockDim.x) {
      const uint32_t key = f32_key(p.v[i]);
      if ((key & mask_hi) == pre0) atomicAdd(&sh[0][(key >> shift) & 255], 1u);
      if (!same && (key & mask_hi) == pre1) atomicAdd(&sh[1][(key >> shift) & 255], 1u);
    }
  }
  __syncthreads();
  if (sh[0][threadIdx.x]) atomicAdd(&p.hist[threadIdx.x], sh[0][threadIdx.x]);
  if (!same && sh[1][threadIdx.x]) atomicAdd(&p.hist[256 + threadIdx.x], sh[1][threadIdx.x]);
}

// One block of 32 threads: walk the histogram(s), fix the next 8 key bits of both targets, clear the histograms.
__global__ void select_decide_kernel(const SelectParams p) {
  if (threadIdx.x < 2) {
    const int t = threadIdx.x;
    const bool same = p.state[2] == p.state[3];
    const unsigned int* h = p.hist + ((same || t == 0) ? 0 : 256);
    unsigned long long rank = p.state[4 + t];
    int b = 0;
    for (; b < 255; ++b) {
      if (rank < h[b]) break;
      rank -= h[b];
    }
    const int shift = 24 - 8 * p.pass;
    const unsigned long long pre = p.state[2 + t] | (static_cast<unsigned long long>(b) << shift);
    __syncwarp(0x3);
    p.state[2 + t] = pre;
    p.state[4 + t] = rank;
    if (p.pass == 3) p.out[t] = key_f32(static_cast<uint32_t>(pre));
  }
  __syncwarp();
  for (int i = threadIdx.x; i < 512; i += 32) p.hist[i] = 0;
  if (p.pass == 3 && threadIdx.x == 0) {
    __threadfence_block();
    const float lo = p.out[0], hi = p.out[1];
    p.out[2] = lo + (hi - lo) * p.frac;          // numpy.percentile(method='linear'): lerp between the neighbours
  }
}

struct ConfMaskParams {
  const float* conf;
  const float* thr;       // device scalar
  unsigned char* mask;
  long long n;
  float floor_;           // conf must also exceed this (0.1 in the reference)
  unsigned long long* count;   // optional: number of kept elements
};

__global__ void __launch_bounds__(256) conf_mask_kernel(const ConfMaskParams p) {
  const float thr = *p.thr;
  unsigned int kept = 0;
  const long long n4 = p.n / 4;
  const float4* c4 = reinterpret_cast<const float4*>(p.conf);
  uchar4* m4 = reinterpret_cast<uchar4*>(p.mask);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n4;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float4 f = c4[i];
    uchar4 m;
    m.x = (f.x >= thr && f.x > p.floor_) ? 1 : 0;
    m.y = (f.y >= thr && f.y > p.floor_) ? 1 : 0;
    m.z = (f.z >= thr && f.z > p.floor_) ? 1 : 0;
    m.w = (f.w >= thr && f.w > p.floor_) ? 1 : 0;
    kept += m.x + m.y + m.z + m.w;
    m4[i] = m;
  }
  if (blockIdx.x == 0) {
    for (long long i = n4 * 4 + threadIdx.x; i < p.n; i += blockDim.x) {
      const float f = p.conf[i];
      const unsigned char m = (f >= thr && f > p.floor_) ? 1 : 0;
      kept += m;
      p.mask[i] = m;
    }
  }
  if (p.count) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) kept += __shfl_xor_sync(0xffffffffu, kept, o);
    if ((threadIdx.x & 31) == 0 && kept) atomicAdd(p.count, static_cast<unsigned long long>(kept));
  }
}

// ---------------------------------------------------------------------------------------------------
// Point cloud (visual_util.py:190-236 predictions_to_glb, inference.py:96-151 viewer): filter, compact, centre, scale.
// Pixels are numbered i = (f * H + y) * W + x, the order of numpy boolean indexing, and compacted as compact.cuh describes:
// cloud_count_kernel, tile_scan_kernel, cloud_gather_kernel.
constexpr int CLOUD_CENTER_BLOCKS = 256;   // fixed, so the fp64 summation order does not depend on the device

struct CloudParams {
  const unsigned char* conf_mask;   // [F*H*W] from conf_mask_kernel
  const float* images;              // [F, 3, H, W] in [0, 1]
  const float* points;              // [F*H*W, 3]
  long long n;                      // F*H*W
  long long hw;                     // H*W
  int black_bg, white_bg, frame0;
  unsigned int* tile_count;         // [tiles]
  unsigned long long* tile_offset;  // [tiles] exclusive prefix of tile_count
  int tiles;                        // compact_tiles(n)
  float* points_out;                // [n_kept, 3]
  unsigned char* colors_out;        // [n_kept, 3]
  int* frame_out;                   // [n_kept]
  float* xyz;                       // [3, ld]: the kept x / y / z as columns (scratch of the scale's percentiles)
  long long ld;
};

// colours as visual_util.py:202 computes them, (x * 255).astype(uint8): fp32 product, truncation (mod 256 like the x86
// conversion numpy uses for values outside [0, 256)), of pixel i of frame f in images fp32 [F, 3, H, W].
__device__ __forceinline__ uchar3 pixel_rgb(const float* images, long long hw, long long i, int f) {
  const float* img = images + f * 2 * hw + i;             // = images + (3 f) hw + (i - f hw)
  uchar3 rgb;
  rgb.x = static_cast<unsigned char>(__float2int_rz(__fmul_rn(img[0], 255.0f)));
  rgb.y = static_cast<unsigned char>(__float2int_rz(__fmul_rn(img[hw], 255.0f)));
  rgb.z = static_cast<unsigned char>(__float2int_rz(__fmul_rn(img[2 * hw], 255.0f)));
  return rgb;
}

// The keep bit of pixel i shared by the point cloud and the mesh: the confidence mask, then the background tests of
// visual_util.py:213-221 on the pixel's colour bytes.
__device__ __forceinline__ bool pixel_keep(const unsigned char* conf_mask, const float* images, long long hw, int black_bg,
                                           int white_bg, long long i, int& f, uchar3& rgb) {
  f = static_cast<int>(i / hw);
  rgb = pixel_rgb(images, hw, i, f);
  bool keep = conf_mask[i] != 0;
  if (black_bg) keep = keep && static_cast<int>(rgb.x) + rgb.y + rgb.z >= 16;
  if (white_bg) keep = keep && !(rgb.x > 240 && rgb.y > 240 && rgb.z > 240);
  return keep;
}

__device__ __forceinline__ bool cloud_keep(const CloudParams& p, long long i, int& f, uchar3& rgb) {
  return pixel_keep(p.conf_mask, p.images, p.hw, p.black_bg, p.white_bg, i, f, rgb);
}

__global__ void __launch_bounds__(COMPACT_THREADS) cloud_count_kernel(const CloudParams p) {
  const long long base = static_cast<long long>(blockIdx.x) * COMPACT_TILE;
  unsigned int kept[1] = {0u};
#pragma unroll 4
  for (int it = 0; it < COMPACT_ITERS; ++it) {
    const long long i = base + it * COMPACT_THREADS + threadIdx.x;
    int f;
    uchar3 rgb;
    if (i < p.n && cloud_keep(p, i, f, rgb)) ++kept[0];
  }
  const unsigned int s = tile_sum<1>(kept);
  if (threadIdx.x == 0) p.tile_count[blockIdx.x] = s;
}

__global__ void __launch_bounds__(COMPACT_THREADS) cloud_gather_kernel(const CloudParams p) {
  const long long base = static_cast<long long>(blockIdx.x) * COMPACT_TILE;
  unsigned long long out = p.tile_offset[blockIdx.x];
  for (int it = 0; it < COMPACT_ITERS; ++it) {
    const long long i = base + it * COMPACT_THREADS + threadIdx.x;
    int f = 0;
    uchar3 rgb = make_uchar3(0, 0, 0);
    const bool keep[1] = {i < p.n && cloud_keep(p, i, f, rgb)};
    unsigned int rank[1], sum[1];
    chunk_ranks<1>(keep, rank, sum);
    if (keep[0]) {
      const unsigned long long k = out + rank[0];
      const float x = p.points[3 * i], y = p.points[3 * i + 1], z = p.points[3 * i + 2];
      p.points_out[3 * k] = x;
      p.points_out[3 * k + 1] = y;
      p.points_out[3 * k + 2] = z;
      p.colors_out[3 * k] = rgb.x;
      p.colors_out[3 * k + 1] = rgb.y;
      p.colors_out[3 * k + 2] = rgb.z;
      p.frame_out[k] = p.frame0 + f;
      p.xyz[k] = x;
      p.xyz[p.ld + k] = y;
      p.xyz[2 * p.ld + k] = z;
    }
    out += sum[0];
  }
}

// Mean of n points (inference.py:111): fp64 partial sums per block in a fixed order, then one thread adds the partials.
struct CloudCenterParams {
  const float* points;   // [n, 3]
  long long n;
  double* partial;       // [CLOUD_CENTER_BLOCKS, 3]
  float* center;         // [3]
};

__global__ void __launch_bounds__(256) cloud_center_partial_kernel(const CloudCenterParams p) {
  __shared__ double sh[3][256];
  double s[3] = {0.0, 0.0, 0.0};
  for (long long i = blockIdx.x * 256LL + threadIdx.x; i < p.n; i += 256LL * CLOUD_CENTER_BLOCKS) {
#pragma unroll
    for (int a = 0; a < 3; ++a) s[a] += static_cast<double>(p.points[3 * i + a]);
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) sh[a][threadIdx.x] = s[a];
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
#pragma unroll
      for (int a = 0; a < 3; ++a) sh[a][threadIdx.x] += sh[a][threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x < 3) p.partial[blockIdx.x * 3 + threadIdx.x] = sh[threadIdx.x][0];
}

__global__ void cloud_center_final_kernel(const CloudCenterParams p) {
  if (threadIdx.x < 3) {
    double s = 0.0;
    for (int b = 0; b < CLOUD_CENTER_BLOCKS; ++b) s += p.partial[b * 3 + threadIdx.x];
    p.center[threadIdx.x] = static_cast<float>(s / static_cast<double>(p.n));
  }
}

// scene_scale = ||p95 - p5|| (visual_util.py:231-236).  sel: the three [lo, hi, interpolated] triples of the 5th percentiles
// (x, y, z) followed by those of the 95th.  fp32 like numpy's norm of a float32 vector.
__global__ void cloud_scale_kernel(const float* sel, float* scale) {
  if (threadIdx.x == 0) {
    float ss = 0.f;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float d = __fsub_rn(sel[(3 + a) * 3 + 2], sel[a * 3 + 2]);
      ss = __fadd_rn(ss, __fmul_rn(d, d));
    }
    *scale = sqrtf(ss);
  }
}

}  // namespace ovg
