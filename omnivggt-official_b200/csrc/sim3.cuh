// Similarity alignment of corresponding point sets, and its application to one view set's predictions (long captures run
// as overlapping view sets, each in its own frame and scale; these kernels put them into one frame).
//   sim3_means_kernel      kept count, sum of src, sum of dst: fp64 partials of a fixed grid
//   sim3_moments_kernel    sum (d - mu_d)(s - mu_s)^T and sum |s - mu_s|^2 about those means: fp64 partials
//   sim3_solve_kernel      one thread: Umeyama (1991) eqs. 40-42 with a one-sided Jacobi SVD of the 3 x 3 covariance
//   sim3_residual_kernel   sum |d - (c R s + t)|^2: fp64 partials; sim3_finish_kernel: the RMS
//   sim3_apply_kernel      points, depth and world-to-camera extrinsics into the target frame, fp64 then rounded once
// Every sum is fp64 in an order fixed by SIM3_BLOCKS and SIM3_THREADS (no float atomics): results are bit-identical from run
// to run and do not depend on the device.
#pragma once
#include <cfloat>

namespace ovg {

constexpr int SIM3_BLOCKS = 256;
constexpr int SIM3_THREADS = 256;
constexpr int SIM3_SWEEPS = 32;      // Jacobi sweeps at most; a 3 x 3 converges in well under 10
enum { SIM3_P0 = 7, SIM3_P1 = 10 };  // doubles per CTA partial of the means / moments passes

struct Sim3Params {
  const float* src;               // [n, 3]
  const float* dst;               // [n, 3]
  const unsigned char* keep;      // [n] or null (all)
  long long n;
  double* part0;                  // [SIM3_BLOCKS][SIM3_P0]: count, sum src (3), sum dst (3)
  double* part1;                  // [SIM3_BLOCKS][SIM3_P1]: sum (d - mu_d)(s - mu_s)^T row-major (9), sum |s - mu_s|^2
  double* part2;                  // [SIM3_BLOCKS]: sum of squared residuals
  double* solved;                 // [12]: c R row-major (9) and t (3), for the residual pass
  double* sim3;                   // [4, 4] out
  double* stats;                  // [4] out: kept count, status, RMS residual, c
};

// Pair i is kept when its keep byte is non-zero and its six coordinates are finite.
__device__ __forceinline__ bool sim3_pair(const Sim3Params& p, long long i, double s[3], double d[3]) {
  if (p.keep && !p.keep[i]) return false;
  bool ok = true;
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const float fs = p.src[3 * i + a], fd = p.dst[3 * i + a];
    ok = ok && isfinite(fs) && isfinite(fd);
    s[a] = fs;
    d[a] = fd;
  }
  return ok;
}

// Sum of each of K per-thread values over the CTA (butterfly within warps, then the warps in order) into out[0..K).
template <int K>
__device__ __forceinline__ void sim3_block_sum(double (&v)[K], double* out) {
  __shared__ double sh[SIM3_THREADS / 32][K];
#pragma unroll
  for (int k = 0; k < K; ++k)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int k = 0; k < K; ++k) sh[threadIdx.x >> 5][k] = v[k];
  __syncthreads();
  if (threadIdx.x < K) {
    double s = 0.0;
    for (int w = 0; w < SIM3_THREADS / 32; ++w) s += sh[w][threadIdx.x];
    out[threadIdx.x] = s;
  }
}

// Column k of the [SIM3_BLOCKS][width] partials, summed over the CTAs in order.
__device__ __forceinline__ double sim3_column(const double* part, int width, int k) {
  double s = 0.0;
  for (int b = 0; b < SIM3_BLOCKS; ++b) s += part[b * width + k];
  return s;
}

__global__ void __launch_bounds__(SIM3_THREADS) sim3_means_kernel(const Sim3Params p) {
  double v[SIM3_P0] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (long long i = blockIdx.x * static_cast<long long>(SIM3_THREADS) + threadIdx.x; i < p.n;
       i += static_cast<long long>(SIM3_THREADS) * SIM3_BLOCKS) {
    double s[3], d[3];
    if (sim3_pair(p, i, s, d)) {
      v[0] += 1.0;
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        v[1 + a] += s[a];
        v[4 + a] += d[a];
      }
    }
  }
  sim3_block_sum<SIM3_P0>(v, p.part0 + blockIdx.x * SIM3_P0);
}

// (kept count, mu_s, mu_d) from the means pass; every CTA and the solver get the same values.
__device__ __forceinline__ void sim3_means(const double (&tot)[SIM3_P0], double& cnt, double ms[3], double md[3]) {
  cnt = tot[0];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    ms[a] = cnt > 0.0 ? tot[1 + a] / cnt : 0.0;
    md[a] = cnt > 0.0 ? tot[4 + a] / cnt : 0.0;
  }
}

__global__ void __launch_bounds__(SIM3_THREADS) sim3_moments_kernel(const Sim3Params p) {
  __shared__ double tot_sh[SIM3_P0];
  if (threadIdx.x < SIM3_P0) tot_sh[threadIdx.x] = sim3_column(p.part0, SIM3_P0, threadIdx.x);
  __syncthreads();
  double tot[SIM3_P0], cnt, ms[3], md[3];
#pragma unroll
  for (int k = 0; k < SIM3_P0; ++k) tot[k] = tot_sh[k];
  sim3_means(tot, cnt, ms, md);
  double v[SIM3_P1] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (long long i = blockIdx.x * static_cast<long long>(SIM3_THREADS) + threadIdx.x; i < p.n;
       i += static_cast<long long>(SIM3_THREADS) * SIM3_BLOCKS) {
    double s[3], d[3];
    if (sim3_pair(p, i, s, d)) {
      const double es[3] = {s[0] - ms[0], s[1] - ms[1], s[2] - ms[2]};
      const double ed[3] = {d[0] - md[0], d[1] - md[1], d[2] - md[2]};
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int c = 0; c < 3; ++c) v[3 * r + c] += ed[r] * es[c];
      v[9] += es[0] * es[0] + es[1] * es[1] + es[2] * es[2];
    }
  }
  sim3_block_sum<SIM3_P1>(v, p.part1 + blockIdx.x * SIM3_P1);
}

// One-sided (Hestenes) Jacobi on the columns of B, accumulating the rotations in V: on return B = U diag(|b_j|) with
// orthogonal columns and B_in = B V^T.  Cyclic pairs (0,1), (0,2), (1,2); a pair is rotated while |b_p . b_q| exceeds
// DBL_EPSILON |b_p| |b_q|; the sweeps stop after the first sweep without a rotation.
__device__ void sim3_jacobi(double B[3][3], double V[3][3]) {
  for (int sweep = 0; sweep < SIM3_SWEEPS; ++sweep) {
    bool rotated = false;
#pragma unroll
    for (int pq = 0; pq < 3; ++pq) {
      const int P = pq == 2 ? 1 : 0, Q = pq == 0 ? 1 : 2;
      double alpha = 0.0, beta = 0.0, gamma = 0.0;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        alpha += B[i][P] * B[i][P];
        beta += B[i][Q] * B[i][Q];
        gamma += B[i][P] * B[i][Q];
      }
      if (!(fabs(gamma) > DBL_EPSILON * sqrt(alpha * beta))) continue;
      const double zeta = (beta - alpha) / (2.0 * gamma);
      const double t = copysign(1.0, zeta) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
      const double c = 1.0 / sqrt(1.0 + t * t), s = c * t;
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const double bp = B[i][P], bq = B[i][Q];
        B[i][P] = c * bp - s * bq;
        B[i][Q] = s * bp + c * bq;
        const double vp = V[i][P], vq = V[i][Q];
        V[i][P] = c * vp - s * vq;
        V[i][Q] = s * vp + c * vq;
      }
      rotated = true;
    }
    if (!rotated) break;
  }
}

__device__ __forceinline__ double det3(const double M[3][3]) {
  return M[0][0] * (M[1][1] * M[2][2] - M[1][2] * M[2][1]) - M[0][1] * (M[1][0] * M[2][2] - M[1][2] * M[2][0]) +
         M[0][2] * (M[1][0] * M[2][1] - M[1][1] * M[2][0]);
}

// Status 0: estimated; 1: fewer than 3 kept pairs; 2: sigma^2 == 0 (all kept src points equal); 3: the second singular
// value of the covariance is not above 1e-12 times the first (collinear or coincident data).  Non-zero: the identity.
__global__ void sim3_solve_kernel(const Sim3Params p) {
  if (threadIdx.x != 0) return;
  double tot[SIM3_P0], cnt, ms[3], md[3];
  for (int k = 0; k < SIM3_P0; ++k) tot[k] = sim3_column(p.part0, SIM3_P0, k);
  sim3_means(tot, cnt, ms, md);
  double mom[SIM3_P1];
  for (int k = 0; k < SIM3_P1; ++k) mom[k] = sim3_column(p.part1, SIM3_P1, k);
  double A[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}}, t[3] = {0.0, 0.0, 0.0}, scale = 1.0;
  int status = 0;
  if (cnt < 3.0) {
    status = 1;
  } else if (mom[9] == 0.0) {
    status = 2;
  } else {
    const double var = mom[9] / cnt;
    double B[3][3], V[3][3] = {{1.0, 0.0, 0.0}, {0.0, 1.0, 0.0}, {0.0, 0.0, 1.0}};
    for (int r = 0; r < 3; ++r)
      for (int c = 0; c < 3; ++c) B[r][c] = mom[3 * r + c] / cnt;
    sim3_jacobi(B, V);
    double sv[3];
    for (int j = 0; j < 3; ++j) sv[j] = sqrt(B[0][j] * B[0][j] + B[1][j] * B[1][j] + B[2][j] * B[2][j]);
    for (int a = 0; a < 2; ++a)            // descending singular values, the columns of B and V with them
      for (int j = 0; j < 2 - a; ++j)
        if (sv[j + 1] > sv[j]) {
          const double x = sv[j]; sv[j] = sv[j + 1]; sv[j + 1] = x;
          for (int i = 0; i < 3; ++i) {
            const double b = B[i][j]; B[i][j] = B[i][j + 1]; B[i][j + 1] = b;
            const double v = V[i][j]; V[i][j] = V[i][j + 1]; V[i][j + 1] = v;
          }
        }
    if (!(sv[1] > 1e-12 * sv[0])) {
      status = 3;
    } else {
      double U[3][3];
      for (int i = 0; i < 3; ++i) {
        U[i][0] = B[i][0] / sv[0];
        U[i][1] = B[i][1] / sv[1];
      }
      // u2 = +-(u0 x u1), the sign that makes B's third column a non-negative multiple of it: exact when the covariance
      // has rank 2 (coplanar points, or N = 3), where b2 / |b2| is not a direction.  R does not depend on that sign.
      double u2[3] = {U[1][0] * U[2][1] - U[2][0] * U[1][1], U[2][0] * U[0][1] - U[0][0] * U[2][1],
                      U[0][0] * U[1][1] - U[1][0] * U[0][1]};
      double d2 = u2[0] * B[0][2] + u2[1] * B[1][2] + u2[2] * B[2][2];
      const double det_u = d2 < 0.0 ? -1.0 : 1.0;
      for (int i = 0; i < 3; ++i) U[i][2] = det_u * u2[i];
      d2 = fabs(d2);
      const double s2 = det_u * det3(V) < 0.0 ? -1.0 : 1.0;       // S = diag(1, 1, s2)
      scale = (sv[0] + sv[1] + s2 * d2) / var;
      for (int r = 0; r < 3; ++r)
        for (int c = 0; c < 3; ++c)
          A[r][c] = scale * (U[r][0] * V[c][0] + U[r][1] * V[c][1] + s2 * U[r][2] * V[c][2]);
      for (int r = 0; r < 3; ++r) t[r] = md[r] - (A[r][0] * ms[0] + A[r][1] * ms[1] + A[r][2] * ms[2]);
    }
  }
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) {
      p.solved[3 * r + c] = A[r][c];
      p.sim3[4 * r + c] = A[r][c];
    }
    p.solved[9 + r] = t[r];
    p.sim3[4 * r + 3] = t[r];
    p.sim3[12 + r] = 0.0;
  }
  p.sim3[15] = 1.0;
  p.stats[0] = cnt;
  p.stats[1] = status;
  p.stats[3] = scale;
}

__global__ void __launch_bounds__(SIM3_THREADS) sim3_residual_kernel(const Sim3Params p) {
  double m[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) m[k] = p.solved[k];
  double v[1] = {0.0};
  for (long long i = blockIdx.x * static_cast<long long>(SIM3_THREADS) + threadIdx.x; i < p.n;
       i += static_cast<long long>(SIM3_THREADS) * SIM3_BLOCKS) {
    double s[3], d[3];
    if (sim3_pair(p, i, s, d)) {
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        const double e = d[r] - (m[3 * r] * s[0] + m[3 * r + 1] * s[1] + m[3 * r + 2] * s[2] + m[9 + r]);
        v[0] += e * e;
      }
    }
  }
  sim3_block_sum<1>(v, p.part2 + blockIdx.x);
}

__global__ void sim3_finish_kernel(const Sim3Params p) {
  if (threadIdx.x == 0) {
    const double ss = sim3_column(p.part2, 1, 0), cnt = p.stats[0];
    p.stats[2] = cnt > 0.0 ? sqrt(ss / cnt) : 0.0;
  }
}

// ---------------------------------------------------------------------------------------------------
// sim3 = [[A, t], [0, 1]] with A = c R.  c = sqrt((A00^2 + A10^2) + A20^2) (the norm of A's first column), R = A / c.
// Every value below is evaluated in fp64 with each product and sum rounded on its own, in the order written (no
// contraction), from the fp32 inputs, and rounded to fp32 once:
//   points      p' = ((A_r0 x + A_r1 y) + A_r2 z) + t_r
//   depth       d' = c d
//   extrinsics  [R_E | t_E] world -> camera:  R'_rj = (R_E,r0 R_j0 + R_E,r1 R_j1) + R_E,r2 R_j2   (R' = R_E R^T),
//               t'_r = c t_E,r - ((R'_r0 t_0 + R'_r1 t_1) + R'_r2 t_2) with R' unrounded
// so unprojecting d' through (K, [R' | t']) gives p' up to fp32 rounding.
struct Sim3ApplyParams {
  const double* sim3;             // [4, 4]
  const float* pts_in[2];         // [n_pix, 3] each, or null
  float* pts_out[2];
  const float* depth_in;          // [n_pix] or null
  float* depth_out;
  const float* ext_in;            // [views, 3, 4] or null
  float* ext_out;
  long long n_pix;
  int views;
};

__device__ __forceinline__ double sim3_dot3(double a0, double a1, double a2, double b0, double b1, double b2) {
  return __dadd_rn(__dadd_rn(__dmul_rn(a0, b0), __dmul_rn(a1, b1)), __dmul_rn(a2, b2));
}

__global__ void __launch_bounds__(256) sim3_apply_kernel(const Sim3ApplyParams p) {
  double A[9], t[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int c = 0; c < 3; ++c) A[3 * r + c] = p.sim3[4 * r + c];
    t[r] = p.sim3[4 * r + 3];
  }
  const double scale = __dsqrt_rn(sim3_dot3(A[0], A[3], A[6], A[0], A[3], A[6]));
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  const long long first = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    if (!p.pts_in[k]) continue;
    const float* in = p.pts_in[k];
    float* out = p.pts_out[k];
    for (long long i = first; i < p.n_pix; i += stride) {
      const double x = in[3 * i], y = in[3 * i + 1], z = in[3 * i + 2];
#pragma unroll
      for (int r = 0; r < 3; ++r)
        out[3 * i + r] = static_cast<float>(__dadd_rn(sim3_dot3(A[3 * r], A[3 * r + 1], A[3 * r + 2], x, y, z), t[r]));
    }
  }
  if (p.depth_in)
    for (long long i = first; i < p.n_pix; i += stride)
      p.depth_out[i] = static_cast<float>(__dmul_rn(scale, static_cast<double>(p.depth_in[i])));
  if (!p.ext_in) return;
  double R[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) R[k] = __ddiv_rn(A[k], scale);
  for (long long v = first; v < p.views; v += stride) {
    const float* e = p.ext_in + v * 12;
    float* o = p.ext_out + v * 12;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      double Rp[3];
#pragma unroll
      for (int j = 0; j < 3; ++j) {
        Rp[j] = sim3_dot3(e[4 * r], e[4 * r + 1], e[4 * r + 2], R[3 * j], R[3 * j + 1], R[3 * j + 2]);
        o[4 * r + j] = static_cast<float>(Rp[j]);
      }
      o[4 * r + 3] = static_cast<float>(
          __dsub_rn(__dmul_rn(scale, static_cast<double>(e[4 * r + 3])), sim3_dot3(Rp[0], Rp[1], Rp[2], t[0], t[1], t[2])));
    }
  }
}

}  // namespace ovg
