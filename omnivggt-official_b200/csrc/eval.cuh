// Scores of one scene's predictions against its ground truth (scene.evaluate): trajectory and pairwise pose errors, depth
// errors after median scaling, and point-map accuracy / completeness / normal consistency.  The reference scores poses only,
// on the host through evo (omnivggt/utils/vo_eval.py:163-246).
//   eval_pose_prep_kernel    one CTA: the views with a camera, their fp64 camera-to-world poses (compacted in view order) and
//                            fp32 centres for the Umeyama fit (sim3.cuh)
//   eval_rpe_kernel          one thread per consecutive pair of the aligned trajectory: evo's RPE with delta = 1
//   eval_pair_kernel         one thread per pair i < j: rotation / translation-direction errors, per-CTA integer histograms
//   eval_pose_finish_kernel  RMS of the RPE, AUC / RRA / RTA from the summed histograms
//   eval_depth_fill_kernel   the valid ground-truth and predicted depths in place, +inf elsewhere, for the two medians
//   eval_depth_partial_kernel / eval_depth_finish_kernel
//                            per-(view, tile) fp64 partials and integer delta counts after median scaling, then per view and
//                            per scene
//   eval_points_keep_kernel  the shared pixel set of both clouds, and the inverse of every ground-truth extrinsic
//   eval_normals_kernel      grid normals of both clouds from the central differences of the pixel grid
//   eval_points_dist_kernel  nearest-neighbour distances and normal dots from the matcher's workspace (match.cuh), both directions
//   eval_points_finish_kernel
// Medians use post.cuh's exact radix selection, its ranks taken from a count on the device (eval_select_init_kernel).  Every
// sum is fp64 over a fixed grid, then in a fixed order, and every count is an integer: results are bit-identical from run to
// run.  No float atomics.
#pragma once
#include "compact.cuh"
#include "match.cuh"
#include "post.cuh"
#include "sim3.cuh"

namespace ovg {

constexpr int EVAL_THREADS = 256;
constexpr int EVAL_PAIR_BLOCKS = 1024;     // grid of the pairwise kernel (grid-stride): the size of its count partials
constexpr int EVAL_DIST_BLOCKS = 512;      // grid of the distance kernel per direction
constexpr int EVAL_MAX_VIEWS = 8192;       // camera views of the pose group: at most 33.5 M pairs
// per-CTA counts of the pairwise kernel: [0, 30) errors in [k, k + 1); 30 + t errors == tau_t; 33 + t RRE < tau_t;
// 36 + t RTE < tau_t
constexpr int EVAL_PAIR_COUNTS = 39;
constexpr int EVAL_DEPTH_P = 7;            // per-(view, tile) partial: sum |sp - g| / g, sum (sp - g)^2 / g, sum (sp - g)^2,
                                           // pixels, delta counts (3)
// the AUC / RRA / RTA thresholds tau_u in degrees
__host__ __device__ constexpr int eval_tau(int u) { return u == 0 ? 5 : (u == 1 ? 10 : 30); }
constexpr double EVAL_DEG = 57.295779513082320876798154814105;   // 180 / pi

// A view has a camera when fx and fy are > 0 and its world-to-camera extrinsic [3, 4] is finite.
__device__ __forceinline__ bool eval_camera_ok(const float* E, const float* K) {
  bool ok = K[0] > 0.f && K[4] > 0.f;
#pragma unroll
  for (int k = 0; k < 12; ++k) ok = ok && isfinite(E[k]);
  return ok;
}

__device__ __forceinline__ bool eval_finite12(const float* E) {
  bool ok = true;
#pragma unroll
  for (int k = 0; k < 12; ++k) ok = ok && isfinite(E[k]);
  return ok;
}

// The rotation angle of R (row-major [9]) in degrees: atan2(|(R21 - R12, R02 - R20, R10 - R01)| / 2, (tr R - 1) / 2).
__device__ __forceinline__ double eval_angle(const double R[9]) {
  const double a = R[7] - R[5], b = R[2] - R[6], c = R[3] - R[1];
  return atan2(sqrt(a * a + b * b + c * c) * 0.5, (R[0] + R[4] + R[8] - 1.0) * 0.5) * EVAL_DEG;
}

// C = A^T B for row-major 3 x 3
__device__ __forceinline__ void eval_atb(const double A[9], const double B[9], double C[9]) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) C[3 * r + c] = A[r] * B[c] + A[3 + r] * B[3 + c] + A[6 + r] * B[6 + c];
}

// --------------------------------------------------------------------------------------------------------------- pose
struct EvalPoseParams {
  const float* gt_ext;            // [S, 3, 4] world -> camera
  const float* gt_intr;           // [S, 3, 3]
  const float* pred_ext;          // [S, 3, 4]
  const int* views;               // [m] scene views to score, distinct, in [0, S)
  int m;
  unsigned char* keep;            // [m] the view has a camera and a finite prediction
  float* centre_gt;               // [m, 3] camera centres -R^T t rounded to fp32, the Umeyama fit's dst
  float* centre_pred;             // [m, 3] its src
  int* count;                     // n: the kept views
  int* vidx;                      // [m] their scene view indices, in order
  double* pose_gt;                // [m][15] the kept views: camera-to-world R^T row-major (9) and centre (3), then t (3)
  double* pose_pred;
  const double* sim3;             // [4, 4] of the fit
  double* rpe;                    // [m][2] per consecutive pair: |t(E)|, angle(R(E))
  unsigned int* pair_counts;      // [EVAL_PAIR_BLOCKS][EVAL_PAIR_COUNTS]
  int* pairs_out;                 // [m (m - 1) / 2, 2]
  double* pair_err;               // [m (m - 1) / 2, 2] RRE, RTE in degrees
  const double* stats;            // the fit's stats: kept count, status, RMS residual (the ATE), c
  double* scores;                 // [12] ate, rpe_trans, rpe_rot, auc (3), rra (3), rta (3)
};

// camera-to-world [R^T | c] in fp64 of a world-to-camera [R | t] fp32, c = -R^T t
__device__ __forceinline__ void eval_c2w(const float* E, double* P) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) P[3 * r + c] = static_cast<double>(E[4 * c + r]);
#pragma unroll
  for (int r = 0; r < 3; ++r)
    P[9 + r] = -(P[3 * r] * static_cast<double>(E[3]) + P[3 * r + 1] * static_cast<double>(E[7]) +
                 P[3 * r + 2] * static_cast<double>(E[11]));
}

// one CTA of 1024 threads
__global__ void __launch_bounds__(1024) eval_pose_prep_kernel(const EvalPoseParams p) {
  for (int k = threadIdx.x; k < p.m; k += 1024) {
    const int v = p.views[k];
    const float* Eg = p.gt_ext + 12LL * v;
    const float* Ep = p.pred_ext + 12LL * v;
    bool ok = eval_camera_ok(Eg, p.gt_intr + 9LL * v) && eval_finite12(Ep);
    double Pg[12], Pp[12];
    eval_c2w(Eg, Pg);
    eval_c2w(Ep, Pp);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const float cg = static_cast<float>(Pg[9 + a]), cp = static_cast<float>(Pp[9 + a]);
      p.centre_gt[3 * k + a] = cg;
      p.centre_pred[3 * k + a] = cp;
      // a finite extrinsic whose centre overflows fp32 would be dropped by the fit (sim3_pair) but not here: drop it here
      ok = ok && isfinite(cg) && isfinite(cp);
    }
    p.keep[k] = ok ? 1 : 0;
  }
  __syncthreads();
  __shared__ int base;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  // ordered compaction, 1024 views per round: ballot ranks within warps, a scan over the warps
  __shared__ int warp_pre[33];
  for (int k0 = 0; k0 < p.m; k0 += 1024) {
    const int k = k0 + threadIdx.x;
    const bool ok = k < p.m && p.keep[k];
    const unsigned int ballot = __ballot_sync(0xffffffffu, ok);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (lane == 0) warp_pre[warp + 1] = __popc(ballot);
    __syncthreads();
    if (threadIdx.x == 0) {
      warp_pre[0] = 0;
      for (int w = 1; w <= 32; ++w) warp_pre[w] += warp_pre[w - 1];
    }
    __syncthreads();
    if (ok) {
      const int q = base + warp_pre[warp] + __popc(ballot & ((1u << lane) - 1u));
      const int v = p.views[k];
      p.vidx[q] = v;
      eval_c2w(p.gt_ext + 12LL * v, p.pose_gt + 15LL * q);
      eval_c2w(p.pred_ext + 12LL * v, p.pose_pred + 15LL * q);
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        p.pose_gt[15LL * q + 12 + r] = p.gt_ext[12LL * v + 4 * r + 3];
        p.pose_pred[15LL * q + 12 + r] = p.pred_ext[12LL * v + 4 * r + 3];
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) base += warp_pre[32];
    __syncthreads();
  }
  if (threadIdx.x == 0) *p.count = base;
}

// grid ceil(m / EVAL_THREADS): pair (k, k + 1) of the kept views (vo_eval.py:201-236, evo's RPE, delta 1 frame, all pairs).
// The prediction after the fit: R_a R, s R_a c + t_a.  E = (Q_k^-1 Q_k+1)^-1 (P_k^-1 P_k+1).
__global__ void __launch_bounds__(EVAL_THREADS) eval_rpe_kernel(const EvalPoseParams p) {
  const int k = blockIdx.x * EVAL_THREADS + threadIdx.x;
  const int n = *p.count;
  if (k + 1 >= n) return;
  double A[9], ta[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int c = 0; c < 3; ++c) A[3 * r + c] = p.sim3[4 * r + c];
    ta[r] = p.sim3[4 * r + 3];
  }
  const double s = sqrt(A[0] * A[0] + A[3] * A[3] + A[6] * A[6]);
  double Ra[9];
#pragma unroll
  for (int e = 0; e < 9; ++e) Ra[e] = A[e] / s;
  double Rq[2][9], cq[2][3], Rp[2][9], cp[2][3];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const double* G = p.pose_gt + 15LL * (k + h);
    const double* P = p.pose_pred + 15LL * (k + h);
#pragma unroll
    for (int e = 0; e < 9; ++e) Rq[h][e] = G[e];
#pragma unroll
    for (int a = 0; a < 3; ++a) cq[h][a] = G[9 + a];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
      for (int c = 0; c < 3; ++c) Rp[h][3 * r + c] = Ra[3 * r] * P[c] + Ra[3 * r + 1] * P[3 + c] + Ra[3 * r + 2] * P[6 + c];
      cp[h][r] = s * (Ra[3 * r] * P[9] + Ra[3 * r + 1] * P[10] + Ra[3 * r + 2] * P[11]) + ta[r];
    }
  }
  // relative motions Q_k^-1 Q_k+1 = [R_k^T R_k+1 | R_k^T (c_k+1 - c_k)], likewise for P
  double Rgr[9], Rpr[9], tgr[3], tpr[3], dq[3], dp[3];
  eval_atb(Rq[0], Rq[1], Rgr);
  eval_atb(Rp[0], Rp[1], Rpr);
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    dq[a] = cq[1][a] - cq[0][a];
    dp[a] = cp[1][a] - cp[0][a];
  }
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    tgr[r] = Rq[0][r] * dq[0] + Rq[0][3 + r] * dq[1] + Rq[0][6 + r] * dq[2];
    tpr[r] = Rp[0][r] * dp[0] + Rp[0][3 + r] * dp[1] + Rp[0][6 + r] * dp[2];
  }
  // E = [Rg^T Rp | Rg^T (tp - tg)]
  double RE[9], d[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) d[a] = tpr[a] - tgr[a];
  eval_atb(Rgr, Rpr, RE);
  double tE2 = 0.0;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double t = Rgr[r] * d[0] + Rgr[3 + r] * d[1] + Rgr[6 + r] * d[2];
    tE2 += t * t;
  }
  p.rpe[2 * k] = sqrt(tE2);
  p.rpe[2 * k + 1] = eval_angle(RE);
}

// The pair (i, j), i < j, of linear index q in the order (0, 1), (0, 2), ..., (1, 2), ...: q = i n - i (i + 1) / 2 + j - i - 1.
__device__ __forceinline__ void eval_pair_ij(long long q, int n, int& i, int& j) {
  const double b = 2.0 * n - 1.0;
  long long ii = static_cast<long long>(floor((b - sqrt(b * b - 8.0 * static_cast<double>(q))) * 0.5));
  if (ii < 0) ii = 0;
  if (ii > n - 2) ii = n - 2;
  auto first = [n](long long r) { return r * n - r * (r + 1) / 2; };
  while (ii > 0 && first(ii) > q) --ii;
  while (ii < n - 2 && first(ii + 1) <= q) ++ii;
  i = static_cast<int>(ii);
  j = static_cast<int>(q - first(ii) + ii + 1);
}

// grid EVAL_PAIR_BLOCKS, grid-stride over the n (n - 1) / 2 pairs.  Relative pose from world-to-camera: R_ij = R_j R_i^T,
// t_ij = t_j - R_ij t_i.  RRE = angle(R_ij,gt^T R_ij,pred); RTE = the angle between t_ij,gt and t_ij,pred folded to
// min(e, 180 - e), 90 when either is zero.
__global__ void __launch_bounds__(EVAL_THREADS) eval_pair_kernel(const EvalPoseParams p) {
  __shared__ unsigned int cnt[EVAL_PAIR_COUNTS];
  for (int c = threadIdx.x; c < EVAL_PAIR_COUNTS; c += EVAL_THREADS) cnt[c] = 0u;
  __syncthreads();
  const int n = *p.count;
  const long long P = static_cast<long long>(n) * (n - 1) / 2;
  for (long long q = blockIdx.x * static_cast<long long>(EVAL_THREADS) + threadIdx.x; q < P;
       q += static_cast<long long>(EVAL_THREADS) * EVAL_PAIR_BLOCKS) {
    int i, j;
    eval_pair_ij(q, n, i, j);
    double R[2][9], t[2][3];
#pragma unroll
    for (int w = 0; w < 2; ++w) {
      const double* Pi = (w ? p.pose_pred : p.pose_gt) + 15LL * i;   // R_i^T, c_i, t_i
      const double* Pj = (w ? p.pose_pred : p.pose_gt) + 15LL * j;
      // R_ij = R_j R_i^T = (R_j^T)^T (R_i^T)
      eval_atb(Pj, Pi, R[w]);
      // from the extrinsics as given (not through c, which would assume R orthonormal to the last bit)
#pragma unroll
      for (int r = 0; r < 3; ++r)
        t[w][r] = Pj[12 + r] - (R[w][3 * r] * Pi[12] + R[w][3 * r + 1] * Pi[13] + R[w][3 * r + 2] * Pi[14]);
    }
    double Rd[9];
    eval_atb(R[0], R[1], Rd);
    const double rre = eval_angle(Rd);
    const double ng = sqrt(t[0][0] * t[0][0] + t[0][1] * t[0][1] + t[0][2] * t[0][2]);
    const double np_ = sqrt(t[1][0] * t[1][0] + t[1][1] * t[1][1] + t[1][2] * t[1][2]);
    double rte = 90.0;
    if (ng > 0.0 && np_ > 0.0) {
      const double cx = t[0][1] * t[1][2] - t[0][2] * t[1][1], cy = t[0][2] * t[1][0] - t[0][0] * t[1][2],
                   cz = t[0][0] * t[1][1] - t[0][1] * t[1][0];
      const double e = atan2(sqrt(cx * cx + cy * cy + cz * cz), t[0][0] * t[1][0] + t[0][1] * t[1][1] + t[0][2] * t[1][2]) * EVAL_DEG;
      rte = fmin(e, 180.0 - e);
    }
    const double err = fmax(rre, rte);
    p.pairs_out[2 * q] = p.vidx[i];
    p.pairs_out[2 * q + 1] = p.vidx[j];
    p.pair_err[2 * q] = rre;
    p.pair_err[2 * q + 1] = rte;
    if (err >= 0.0 && err < 30.0) atomicAdd(&cnt[static_cast<int>(err)], 1u);
#pragma unroll
    for (int u = 0; u < 3; ++u) {
      const double tau = eval_tau(u);
      if (err == tau) atomicAdd(&cnt[30 + u], 1u);
      if (rre < tau) atomicAdd(&cnt[33 + u], 1u);
      if (rte < tau) atomicAdd(&cnt[36 + u], 1u);
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < EVAL_PAIR_COUNTS; c += EVAL_THREADS)
    p.pair_counts[blockIdx.x * EVAL_PAIR_COUNTS + c] = cnt[c];
}

// numpy's pairwise sum of a[0, n) for n <= 128 (eight accumulators, then the remainder in order), so that
// mean(cumsum(hist) / P) is numpy's to the bit
__device__ double eval_numpy_sum(const double* a, int n) {
  if (n < 8) {
    double s = 0.0;
    for (int i = 0; i < n; ++i) s = __dadd_rn(s, a[i]);
    return s;
  }
  double r[8];
  for (int k = 0; k < 8; ++k) r[k] = a[k];
  int i = 8;
  for (; i < n - (n % 8); i += 8)
    for (int k = 0; k < 8; ++k) r[k] = __dadd_rn(r[k], a[i + k]);
  double s = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])), __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; i < n; ++i) s = __dadd_rn(s, a[i]);
  return s;
}

// one CTA of EVAL_THREADS
__global__ void __launch_bounds__(EVAL_THREADS) eval_pose_finish_kernel(const EvalPoseParams p) {
  __shared__ unsigned long long tot[EVAL_PAIR_COUNTS];
  for (int c = threadIdx.x; c < EVAL_PAIR_COUNTS; c += EVAL_THREADS) {
    unsigned long long s = 0;
    for (int b = 0; b < EVAL_PAIR_BLOCKS; ++b) s += p.pair_counts[b * EVAL_PAIR_COUNTS + c];
    tot[c] = s;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  const int n = *p.count;
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  double st = 0.0, sr = 0.0;
  for (int k = 0; k + 1 < n; ++k) {
    st = __dadd_rn(st, __dmul_rn(p.rpe[2 * k], p.rpe[2 * k]));
    sr = __dadd_rn(sr, __dmul_rn(p.rpe[2 * k + 1], p.rpe[2 * k + 1]));
  }
  p.scores[0] = p.stats[2];
  p.scores[1] = n >= 2 ? sqrt(st / (n - 1)) : nan;
  p.scores[2] = n >= 2 ? sqrt(sr / (n - 1)) : nan;
  const double P = static_cast<double>(static_cast<long long>(n) * (n - 1) / 2);
  for (int u = 0; u < 3; ++u) {
    const int tau = eval_tau(u);
    double frac[30];
    unsigned long long cum = 0;
    for (int k = 0; k < tau; ++k) {
      cum += tot[k];
      frac[k] = __ddiv_rn(static_cast<double>(k + 1 == tau ? cum + tot[30 + u] : cum), P);
    }
    p.scores[3 + u] = P > 0.0 ? __ddiv_rn(eval_numpy_sum(frac, tau), static_cast<double>(tau)) : nan;
    p.scores[6 + u] = P > 0.0 ? __ddiv_rn(static_cast<double>(tot[33 + u]), P) : nan;
    p.scores[9 + u] = P > 0.0 ? __ddiv_rn(static_cast<double>(tot[36 + u]), P) : nan;
  }
}

// ---------------------------------------------------------------------------------------------------- medians on a count
// select_init_kernel with n read from the device (0 selects nothing: both ranks 0)
__global__ void eval_select_init_kernel(unsigned long long* state, unsigned int* hist, const unsigned long long* count,
                                        float percent, float* weight) {
  if (threadIdx.x == 0) select_init_ranks(static_cast<long long>(*count), percent, state, weight);
  for (int i = threadIdx.x; i < 512; i += blockDim.x) hist[i] = 0;
}

// --------------------------------------------------------------------------------------------------------------- depth
struct EvalDepthParams {
  const float* gt;                // [S, H W]
  const unsigned char* mask;      // [S, H W] or null (every pixel)
  const float* pred;              // [S, H W]
  const unsigned char* view_sel;  // [S]
  int S;
  long long hw;
  int tiles;                      // tiles of COMPACT_TILE pixels per view
  long long ld;                   // column stride of cols
  float* cols;                    // [2, ld] valid g, valid p, +inf elsewhere
  unsigned long long* count;      // valid pixels
  float* sel;                     // [2][3] selection results (lo, hi) of g and p
  float* weight;                  // [2] their weights
  double* part;                   // [S, tiles, EVAL_DEPTH_P]
  double* view_tot;               // [S, EVAL_DEPTH_P]
  double* scores;                 // [10] pixels, scale, median g, median p, abs_rel, sq_rel, rmse, delta (3)
  double* view_abs_rel;           // [S]
  double* view_delta1;            // [S]
  long long* view_pixels;         // [S]
};

__device__ __forceinline__ bool eval_depth_valid(const EvalDepthParams& p, long long i, float& g, float& d) {
  if (!p.view_sel[i / p.hw] || (p.mask && !p.mask[i])) return false;
  g = p.gt[i];
  d = p.pred[i];
  return g > 0.f && isfinite(g) && isfinite(d);
}

__global__ void __launch_bounds__(EVAL_THREADS) eval_depth_fill_kernel(const EvalDepthParams p) {
  const long long n = static_cast<long long>(p.S) * p.hw;
  unsigned int kept = 0;
  for (long long i = blockIdx.x * static_cast<long long>(EVAL_THREADS) + threadIdx.x; i < p.ld;
       i += static_cast<long long>(EVAL_THREADS) * gridDim.x) {
    float g = 0.f, d = 0.f;
    const bool ok = i < n && eval_depth_valid(p, i, g, d);
    p.cols[i] = ok ? g : __int_as_float(0x7f800000);
    p.cols[p.ld + i] = ok ? d : __int_as_float(0x7f800000);
    kept += ok;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) kept += __shfl_xor_sync(0xffffffffu, kept, o);
  if ((threadIdx.x & 31) == 0 && kept) atomicAdd(p.count, static_cast<unsigned long long>(kept));
}

// scale = median(g) / median(p) in fp64, each median numpy.percentile(v, 50) of the fp32 values
__device__ __forceinline__ double eval_depth_scale(const EvalDepthParams& p, float& mg, float& mp) {
  mg = select_lerp(p.sel[0], p.sel[1], p.weight[0]);
  mp = select_lerp(p.sel[3], p.sel[4], p.weight[1]);
  return __ddiv_rn(static_cast<double>(mg), static_cast<double>(mp));
}

// grid (tiles, min(S, 65535)): the y blocks stride over the views, so any S launches; each (view, tile) partial is the same
__global__ void __launch_bounds__(EVAL_THREADS) eval_depth_partial_kernel(const EvalDepthParams p) {
  float mg, mp;
  const double s = eval_depth_scale(p, mg, mp);
  const long long base = static_cast<long long>(blockIdx.x) * COMPACT_TILE;
  for (int v = blockIdx.y; v < p.S; v += gridDim.y) {
    double acc[EVAL_DEPTH_P] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int it = 0; it < COMPACT_ITERS; ++it) {
      const long long i = base + it * COMPACT_THREADS + threadIdx.x;
      float g, d;
      if (i < p.hw && eval_depth_valid(p, v * p.hw + i, g, d)) {
        const double gd = g, sp = __dmul_rn(s, static_cast<double>(d)), e = __dsub_rn(sp, gd), e2 = __dmul_rn(e, e);
        acc[0] = __dadd_rn(acc[0], __ddiv_rn(fabs(e), gd));
        acc[1] = __dadd_rn(acc[1], __ddiv_rn(e2, gd));
        acc[2] = __dadd_rn(acc[2], e2);
        acc[3] += 1.0;
        const double r = fmax(__ddiv_rn(sp, gd), __ddiv_rn(gd, sp));
        acc[4] += r < 1.25 ? 1.0 : 0.0;
        acc[5] += r < 1.5625 ? 1.0 : 0.0;
        acc[6] += r < 1.953125 ? 1.0 : 0.0;
      }
    }
    sim3_block_sum<EVAL_DEPTH_P>(acc, p.part + (static_cast<long long>(v) * p.tiles + blockIdx.x) * EVAL_DEPTH_P);
    __syncthreads();                // the block sum's shared partials are read before the next view writes them
  }
}

// one CTA of EVAL_THREADS: each view's tiles in order, then the views in order
__global__ void __launch_bounds__(EVAL_THREADS) eval_depth_finish_kernel(const EvalDepthParams p) {
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  for (int v = threadIdx.x; v < p.S; v += EVAL_THREADS) {
    double t[EVAL_DEPTH_P] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int b = 0; b < p.tiles; ++b)
      for (int k = 0; k < EVAL_DEPTH_P; ++k) t[k] = __dadd_rn(t[k], p.part[(static_cast<long long>(v) * p.tiles + b) * EVAL_DEPTH_P + k]);
    for (int k = 0; k < EVAL_DEPTH_P; ++k) p.view_tot[static_cast<long long>(v) * EVAL_DEPTH_P + k] = t[k];
    p.view_pixels[v] = static_cast<long long>(t[3]);
    p.view_abs_rel[v] = t[3] > 0.0 ? __ddiv_rn(t[0], t[3]) : nan;
    p.view_delta1[v] = t[3] > 0.0 ? __ddiv_rn(t[4], t[3]) : nan;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double t[EVAL_DEPTH_P] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int v = 0; v < p.S; ++v)
    for (int k = 0; k < EVAL_DEPTH_P; ++k) t[k] = __dadd_rn(t[k], p.view_tot[static_cast<long long>(v) * EVAL_DEPTH_P + k]);
  const double n = t[3];
  float mg, mp;
  const double s = eval_depth_scale(p, mg, mp);
  p.scores[0] = n;
  p.scores[1] = n > 0.0 ? s : nan;
  p.scores[2] = n > 0.0 ? static_cast<double>(mg) : nan;
  p.scores[3] = n > 0.0 ? static_cast<double>(mp) : nan;
  p.scores[4] = n > 0.0 ? __ddiv_rn(t[0], n) : nan;
  p.scores[5] = n > 0.0 ? __ddiv_rn(t[1], n) : nan;
  p.scores[6] = n > 0.0 ? __dsqrt_rn(__ddiv_rn(t[2], n)) : nan;
  for (int k = 0; k < 3; ++k) p.scores[7 + k] = n > 0.0 ? __ddiv_rn(t[4 + k], n) : nan;
}

// -------------------------------------------------------------------------------------------------------------- points
struct EvalKeepParams {
  const float* gt_ext;            // [S, 3, 4]
  const float* gt_intr;           // [S, 3, 3]
  const float* gt_depth;          // [S, H W]
  const unsigned char* mask;      // [S, H W] or null
  const float* pred_points;       // [S, H W, 3]
  const unsigned char* view_sel;  // [S]
  int S;
  long long hw;
  float* c2w;                     // [S, 3, 4] out: [R^T | -R^T t], fp64 then rounded once
  unsigned char* keep;            // [2, S H W] out: the shared pixel set, once per cloud
};

// grid-stride over the S H W pixels; the first S threads also invert the extrinsics (closed_form_inverse_se3)
__global__ void __launch_bounds__(EVAL_THREADS) eval_points_keep_kernel(const EvalKeepParams p) {
  const long long n = static_cast<long long>(p.S) * p.hw;
  const long long first = blockIdx.x * static_cast<long long>(EVAL_THREADS) + threadIdx.x;
  const long long stride = static_cast<long long>(EVAL_THREADS) * gridDim.x;
  for (long long v = first; v < p.S; v += stride) {
    double P[12];
    eval_c2w(p.gt_ext + 12 * v, P);
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
      for (int c = 0; c < 3; ++c) p.c2w[12 * v + 4 * r + c] = static_cast<float>(P[3 * r + c]);
      p.c2w[12 * v + 4 * r + 3] = static_cast<float>(P[9 + r]);
    }
  }
  for (long long i = first; i < n; i += stride) {
    const long long v = i / p.hw;
    bool ok = p.view_sel[v] && (!p.mask || p.mask[i]) && eval_camera_ok(p.gt_ext + 12 * v, p.gt_intr + 9 * v);
    const float g = p.gt_depth[i];
    ok = ok && g > 0.f && isfinite(g);
#pragma unroll
    for (int a = 0; a < 3; ++a) ok = ok && isfinite(p.pred_points[3 * i + a]);
    p.keep[i] = ok ? 1 : 0;
    p.keep[n + i] = ok ? 1 : 0;
  }
}

struct EvalPointsParams {
  MatchParams m;                  // the matcher's workspace over V = 2 views (0: aligned prediction, 1: ground truth) and the
                                  // one pair (0, 1): pts, grid[v].n, nn
  const float* points;            // [2, S H W, 3] the clouds the matcher indexed
  const unsigned char* keep;      // [2, S H W]
  int S, H, W;
  double* normals;                // [2, S H W, 3]; NaN x: no normal
  long long ld;                   // column stride of cols
  float* cols;                    // [2, ld] distances rounded to fp32, +inf past the kept count
  unsigned long long* count;      // [2] kept counts, for the medians
  double* part;                   // [2, EVAL_DIST_BLOCKS, 3]: sum of distances, sum of |n . n_nn|, pairs with both normals
  float* sel;                     // [2][3] median selections
  float* weight;                  // [2]
  double* dist[2];                // [n] out: accuracy (prediction -> ground truth), completeness (ground truth -> prediction)
  double* scores;                 // [9] pixels, acc, acc_median, comp, comp_median, chamfer, nc_acc, nc_comp, nc
};

__device__ __forceinline__ bool eval_kept(const EvalPointsParams& p, int c, int v, int y, int x) {
  return y >= 0 && y < p.H && x >= 0 && x < p.W &&
         p.keep[static_cast<long long>(c) * p.S * p.H * p.W + (static_cast<long long>(v) * p.H + y) * p.W + x];
}

// grid-stride over both clouds: n = normalize((P[x+1, y] - P[x-1, y]) x (P[x, y+1] - P[x, y-1])) when the pixel and its four
// neighbours are in the set and the cross product is not zero; every operation fp64, rounded on its own
__global__ void __launch_bounds__(EVAL_THREADS) eval_normals_kernel(const EvalPointsParams p) {
  const long long hw = static_cast<long long>(p.H) * p.W, n = p.S * hw;
  for (long long e = blockIdx.x * static_cast<long long>(EVAL_THREADS) + threadIdx.x; e < 2 * n;
       e += static_cast<long long>(EVAL_THREADS) * gridDim.x) {
    const int c = e >= n ? 1 : 0;
    const long long i = e - c * n;
    const int v = static_cast<int>(i / hw), y = static_cast<int>((i % hw) / p.W), x = static_cast<int>(i % p.W);
    double* out = p.normals + 3 * e;
    double nx = __longlong_as_double(0x7ff8000000000000LL), ny = 0.0, nz = 0.0;
    if (eval_kept(p, c, v, y, x) && eval_kept(p, c, v, y, x - 1) && eval_kept(p, c, v, y, x + 1) &&
        eval_kept(p, c, v, y - 1, x) && eval_kept(p, c, v, y + 1, x)) {
      const float* P = p.points + 3 * (c * n);
      const float* xr = P + 3 * (i + 1);
      const float* xl = P + 3 * (i - 1);
      const float* yd = P + 3 * (i + p.W);
      const float* yu = P + 3 * (i - p.W);
      double a[3], b[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        a[k] = __dsub_rn(static_cast<double>(xr[k]), static_cast<double>(xl[k]));
        b[k] = __dsub_rn(static_cast<double>(yd[k]), static_cast<double>(yu[k]));
      }
      const double cx = __dsub_rn(__dmul_rn(a[1], b[2]), __dmul_rn(a[2], b[1]));
      const double cy = __dsub_rn(__dmul_rn(a[2], b[0]), __dmul_rn(a[0], b[2]));
      const double cz = __dsub_rn(__dmul_rn(a[0], b[1]), __dmul_rn(a[1], b[0]));
      const double len = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(cx, cx), __dmul_rn(cy, cy)), __dmul_rn(cz, cz)));
      if (len > 0.0) {
        nx = __ddiv_rn(cx, len);
        ny = __ddiv_rn(cy, len);
        nz = __ddiv_rn(cz, len);
      }
    }
    out[0] = nx;
    out[1] = ny;
    out[2] = nz;
  }
}

// grid (EVAL_DIST_BLOCKS, 2): direction c queries cloud c against cloud 1 - c (matcher segment c of pair (0, 1)).  The distance
// is sqrt of the matcher's fp64 d2 = ((dx dx) + (dy dy)) + dz dz; the normal dot |n . n_nn| counts when both have a normal.
__global__ void __launch_bounds__(EVAL_THREADS) eval_points_dist_kernel(const EvalPointsParams p) {
  const int c = blockIdx.y;
  const long long cap = p.m.cap;
  const int nq = p.m.grid[c].n;
  double acc[3] = {0.0, 0.0, 0.0};
  for (long long k = blockIdx.x * static_cast<long long>(EVAL_THREADS) + threadIdx.x; k < p.ld;
       k += static_cast<long long>(EVAL_THREADS) * EVAL_DIST_BLOCKS) {
    if (k >= nq) {
      p.cols[c * p.ld + k] = __int_as_float(0x7f800000);
      continue;
    }
    const float4 q = p.m.pts[c * cap + k];
    const int nn = p.m.nn[c * cap + k];
    double d = __longlong_as_double(0x7ff8000000000000LL);
    if (nn >= 0) {
      const float4 t = p.m.pts[(1 - c) * cap + nn];
      const double dx = __dsub_rn(static_cast<double>(q.x), static_cast<double>(t.x));
      const double dy = __dsub_rn(static_cast<double>(q.y), static_cast<double>(t.y));
      const double dz = __dsub_rn(static_cast<double>(q.z), static_cast<double>(t.z));
      d = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
      const double* a = p.normals + 3 * (c * cap + __float_as_int(q.w));
      const double* b = p.normals + 3 * ((1 - c) * cap + __float_as_int(t.w));
      if (!isnan(a[0]) && !isnan(b[0])) {
        acc[1] = __dadd_rn(acc[1], fabs(__dadd_rn(__dadd_rn(__dmul_rn(a[0], b[0]), __dmul_rn(a[1], b[1])), __dmul_rn(a[2], b[2]))));
        acc[2] += 1.0;
      }
    }
    acc[0] = __dadd_rn(acc[0], d);
    p.dist[c][k] = d;
    p.cols[c * p.ld + k] = static_cast<float>(d);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) p.count[c] = static_cast<unsigned long long>(nq);
  sim3_block_sum<3>(acc, p.part + (c * EVAL_DIST_BLOCKS + blockIdx.x) * 3);
}

__global__ void eval_points_finish_kernel(const EvalPointsParams p) {
  if (threadIdx.x != 0) return;
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  double t[2][3];
  for (int c = 0; c < 2; ++c)
    for (int k = 0; k < 3; ++k) {
      double s = 0.0;
      for (int b = 0; b < EVAL_DIST_BLOCKS; ++b) s = __dadd_rn(s, p.part[(c * EVAL_DIST_BLOCKS + b) * 3 + k]);
      t[c][k] = s;
    }
  const double n = static_cast<double>(p.count[0]);
  const double acc = n > 0.0 ? __ddiv_rn(t[0][0], n) : nan, comp = n > 0.0 ? __ddiv_rn(t[1][0], n) : nan;
  const double nca = t[0][2] > 0.0 ? __ddiv_rn(t[0][1], t[0][2]) : nan, ncc = t[1][2] > 0.0 ? __ddiv_rn(t[1][1], t[1][2]) : nan;
  p.scores[0] = n;
  p.scores[1] = acc;
  p.scores[2] = n > 0.0 ? static_cast<double>(select_lerp(p.sel[0], p.sel[1], p.weight[0])) : nan;
  p.scores[3] = comp;
  p.scores[4] = n > 0.0 ? static_cast<double>(select_lerp(p.sel[3], p.sel[4], p.weight[1])) : nan;
  p.scores[5] = __dmul_rn(__dadd_rn(acc, comp), 0.5);
  p.scores[6] = nca;
  p.scores[7] = ncc;
  p.scores[8] = __dmul_rn(__dadd_rn(nca, ncc), 0.5);
}

}  // namespace ovg
