// Bundle adjustment of a scene's tracks (ovg_bundle_adjust): Levenberg-Marquardt over the views' poses and focal lengths and
// the track points, the points eliminated by a Schur complement and the reduced camera system solved by preconditioned
// conjugate gradients (Wu et al., "Multicore Bundle Adjustment", CVPR 2011; Ceres' ITERATIVE_SCHUR).  No counterpart in the
// reference; the conventions are COLMAP's PINHOLE bundle adjustment.
//   ba_init_kernel          one thread: LM state, fp64 cameras, the gauge (view 0's pose, view 1's largest baseline
//                           coordinate) as a per-view parameter mask
//   ba_track_init_kernel    per track: the observations' track, the starting point, whether the track is refined
//   ba_view_count_kernel    \  per view, the stable ordered compaction of the observations (compact.cuh): each view's
//   ba_view_gather_kernel   /  observations in observation order
//   ba_eval_kernel          per track: cost at the current or the trial point, model decrease, step and parameter norms,
//                           fp64 partials per block
//   ba_control_kernel       one block, one deciding thread: accept / reject, mu, nu, the stop rules, the counters
//   ba_track_kernel         per track: Jacobians (after an accepted step), V_p + D_p / mu inverted, V_p^-1 g_p
//   ba_view_block_kernel    per view and chunk: partial sums of U_v, W V^-1 W^T, g_v and W V^-1 g_p
//   ba_view_reduce_kernel   per view: those chunk partials summed in order
//   ba_pcg_kernel           one cooperative launch: block-Jacobi PCG on S dc = b with S applied implicitly, then the
//                           back-substitution of the points and the trial cameras
//   ba_output_kernel        per track: refined point and reprojection error (track_reproject, as track_point_kernel)
//   ba_finish_kernel        cameras, cost and counters
// Every fp64 sum has a fixed grid and a fixed order (per-block or per-chunk partials, then an in-order reduction), the
// cooperative kernel's CTAs each repeat the per-view arithmetic on identical data, and no float atomic is used: results are
// bit-identical from run to run.  After a stop every later kernel returns at once.
#pragma once
#include "fps.cuh"
#include "tracks.cuh"

namespace ovg {

constexpr int BA_THREADS = 128;         // per-track kernels
constexpr int BA_CAM = 21;              // doubles per camera: [R | t] row-major (12), K row-major (9)
constexpr int BA_NP = 8;                // parameters per view: rotation increment (3), translation (3), fx, fy
constexpr int BA_PACK = 36;             // packed lower triangle of an 8 x 8 block
constexpr int BA_ENTRIES = 88;          // per-view sums: U (36), W V^-1 W^T (36), g (8), W V^-1 g_p (8)
constexpr int BA_BLOCK_CHUNKS = 64;     // chunks per view of ba_view_block_kernel
constexpr int BA_BLOCK_BATCH = 32;      // observations staged in shared memory at a time
constexpr int BA_BLOCK_THREADS = 96;
constexpr int BA_OBS_DOUBLES = 26;      // sizeof(BaObs) / 8
constexpr int BA_STAGE = 37;            // staged doubles per observation: BaObs up to w (25), V_p^-1 (9), V_p^-1 g_p (3)
constexpr int BA_PCG_CHUNKS = 32;       // chunks per view of the PCG's per-view pass
constexpr int BA_PCG_THREADS = 256;
constexpr int BA_PCG_MAX = 500;
constexpr int BA_MAX_VIEWS = BA_PCG_THREADS;   // one view per thread in the PCG's per-view steps
constexpr int BA_VIEW_SMEM = 104;       // doubles per view in the PCG's shared memory: U*, L (36 each), x, r, p, q / z (8 each)
constexpr int BA_EVAL = 6;              // per-block sums of ba_eval_kernel

struct BaObs {                          // one observation at the current linearisation
  double jc[2][BA_NP];                  // d residual / d camera parameters, fixed parameters' columns zero
  double jp[2][3];                      // d residual / d point
  double r[2];                          // residual
  double w;                             // IRLS weight rho'(|r|^2); 0 for an observation of a track that is not refined
  double pad;
};
static_assert(sizeof(BaObs) == BA_OBS_DOUBLES * 8, "BaObs layout");

struct BaState {
  double mu, nu, cost;                  // LM radius and its growth, current cost 1/2 sum rho
  double cam_step2, cam_x2;             // camera parts of |delta|^2 and |x|^2 (ba_pcg_kernel)
  long long steps, accepted, pcg;
  int cur, stop, status, lin, small, its;   // current parameter buffer, stopped, status, relinearise, |g|inf small, PCG its
  unsigned arrive;                      // grid barrier of ba_pcg_kernel, zeroed by ba_control_kernel
};

struct BaParams {
  int V, iterations, refine_focal, cauchy;
  long long n, m;
  int tblocks;                          // ceil(n / BA_THREADS), at least 1
  int vtiles;                           // compact_tiles(m), at least 1
  double c2;                            // loss_scale^2
  const double* points;                 // [n, 3]
  const long long* offsets;             // [n + 1]
  const int* view;                      // [m]
  const double* obs;                    // [m, 2] COLMAP pixel frame
  const float* ext;                     // [V, 3, 4]
  const float* intr;                    // [V, 3, 3]
  // workspace
  BaState* st;
  double* cam;                          // [2][V][BA_CAM] current and trial
  double* mask;                         // [V][BA_NP] 1 free, 0 fixed
  double* dcam;                         // [V][BA_NP] camera step
  double* pts;                          // [2][n][3] current and trial
  double* dp;                           // [n][3] point step
  double* vinv;                         // [n][9] (V_p + D_p / mu)^-1
  double* y;                            // [n][3] V_p^-1 g_p
  double* gp;                           // [n][3] g_p
  double* zt;                           // [n][3] PCG: V_p^-1 sum W^T p
  unsigned char* incl;                  // [n] refined track
  BaObs* ob;                            // [m]
  int* obs_track;                       // [m]
  int* view_obs;                        // [m] observations by view, observation order within a view
  long long* view_off;                  // [V + 1]
  double* gmax;                         // [tblocks] max |g_p| per block
  double* vpart;                        // [V][BA_BLOCK_CHUNKS][BA_ENTRIES]
  double* vsum;                         // [V][BA_ENTRIES]
  double* bpart;                        // [V][BA_PCG_CHUNKS][BA_NP]
  double* epart;                        // [tblocks][BA_EVAL]
  unsigned int* tile_count;             // [V][vtiles]
  unsigned long long* tile_offset;      // [V][vtiles]
  unsigned long long* scan_total;
  // outputs
  double* points_out;                   // [n, 3]
  double* ext_out;                      // [V, 3, 4]
  double* intr_out;                     // [V, 3, 3]
  double* error_out;                    // [n]
  double* cost_out;                     // [2]
  long long* stats_out;                 // [4] steps, accepted, PCG iterations, status
  double* trace;                        // [iterations] cost after each step, or null
};

__host__ __device__ constexpr int ba_pk(int i, int j) { return i * (i + 1) / 2 + j; }   // i >= j

__device__ __forceinline__ double ba_rho(const BaParams& p, double s) { return p.cauchy ? p.c2 * log1p(s / p.c2) : s; }
__device__ __forceinline__ double ba_weight(const BaParams& p, double s) { return p.cauchy ? 1.0 / (1.0 + s / p.c2) : 1.0; }
__device__ __forceinline__ double ba_clamp(double d) { return fmin(fmax(d, 1e-6), 1e32); }

// Fixed-order sum of one value per thread over a block of BA_PCG_THREADS (or fewer, whole warps); every thread gets it.
template <int T>
__device__ __forceinline__ double ba_block_sum(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);   // every lane ends with the same bits
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int w = 0; w < T / 32; ++w) s += red[w];
  __syncthreads();
  return s;
}

template <int T>
__device__ __forceinline__ double ba_block_max(double v, double* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int w = 0; w < T / 32; ++w) s = fmax(s, red[w]);
  __syncthreads();
  return s;
}

__device__ __forceinline__ void ba_obs_range(const BaParams& p, long long t, long long& b, long long& e) {
  b = p.offsets[t];
  e = p.offsets[t + 1];
}

// ---------------------------------------------------------------------------------------------------------------- set-up
__global__ void ba_init_kernel(const BaParams p) {
  BaState* s = p.st;
  s->mu = 1e4; s->nu = 2.0; s->cost = 0.0; s->cam_step2 = 0.0; s->cam_x2 = 0.0;
  s->steps = 0; s->accepted = 0; s->pcg = 0;
  s->cur = 0; s->stop = 0; s->status = 1; s->lin = 1; s->small = 0; s->its = 0; s->arrive = 0u;
  for (int v = 0; v < p.V; ++v) {
#pragma unroll
    for (int i = 0; i < 12; ++i) p.cam[v * BA_CAM + i] = p.ext[12 * v + i];
#pragma unroll
    for (int i = 0; i < 9; ++i) p.cam[v * BA_CAM + 12 + i] = p.intr[9 * v + i];
  }
  // the gauge: t1 - R1 R0^T t0, the baseline in camera 1; its largest coordinate (the first on ties) is held
  const float* E0 = p.ext;
  const float* E1 = p.ext + 12;
  double c[3];
#pragma unroll
  for (int a = 0; a < 3; ++a)
    c[a] = static_cast<double>(E0[a]) * E0[3] + static_cast<double>(E0[4 + a]) * E0[7] + static_cast<double>(E0[8 + a]) * E0[11];
  int k = 0;
  double best = -1.0;                                          // |d_r| of the held coordinate so far
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const double d = static_cast<double>(E1[4 * r + 3]) -
                     (static_cast<double>(E1[4 * r]) * c[0] + static_cast<double>(E1[4 * r + 1]) * c[1] +
                      static_cast<double>(E1[4 * r + 2]) * c[2]);
    if (fabs(d) > best) {
      best = fabs(d);
      k = r;
    }
  }
  for (int v = 0; v < p.V; ++v)
#pragma unroll
    for (int i = 0; i < BA_NP; ++i) {
      const bool fixed = (v == 0 && i < 6) || (v == 1 && i == 3 + k) || (i >= 6 && !p.refine_focal);
      p.mask[v * BA_NP + i] = fixed ? 0.0 : 1.0;
    }
  if (p.trace)
    for (int i = 0; i < p.iterations; ++i) p.trace[i] = __longlong_as_double(0x7ff8000000000000LL);
}

// per track: a track is refined when it has two observations or more and every camera sees its start in front
__global__ void __launch_bounds__(BA_THREADS) ba_track_init_kernel(const BaParams p) {
  const long long t = static_cast<long long>(blockIdx.x) * BA_THREADS + threadIdx.x;
  if (t >= p.n) return;
  long long b, e;
  ba_obs_range(p, t, b, e);
  const double c[3] = {p.points[3 * t], p.points[3 * t + 1], p.points[3 * t + 2]};
  bool behind = false;
  for (long long q = b; q < e; ++q) {
    p.obs_track[q] = static_cast<int>(t);
    const double* C = p.cam + p.view[q] * BA_CAM;
    double X[3], du, dv;
    behind |= track_reproject(C, C + 12, c, p.obs[2 * q], p.obs[2 * q + 1], X, du, dv);
  }
#pragma unroll
  for (int a = 0; a < 3; ++a) p.pts[3 * t + a] = c[a];
  p.incl[t] = (e - b >= 2 && !behind) ? 1 : 0;
}

// grid (vtiles, V): observations of view v per tile
__global__ void __launch_bounds__(COMPACT_THREADS) ba_view_count_kernel(const BaParams p) {
  const int v = blockIdx.y;
  const long long base = static_cast<long long>(blockIdx.x) * COMPACT_TILE;
  unsigned int c[1] = {0u};
  for (int it = 0; it < COMPACT_ITERS; ++it) {
    const long long o = base + it * COMPACT_THREADS + threadIdx.x;
    c[0] += (o < p.m && p.view[o] == v) ? 1u : 0u;
  }
  const unsigned int s = tile_sum<1>(c);
  if (threadIdx.x == 0) p.tile_count[v * p.vtiles + blockIdx.x] = s;
}

// grid (vtiles, V), after the scan of the tile counts
__global__ void __launch_bounds__(COMPACT_THREADS) ba_view_gather_kernel(const BaParams p) {
  const int v = blockIdx.y;
  const long long base = static_cast<long long>(blockIdx.x) * COMPACT_TILE;
  unsigned long long out = p.tile_offset[static_cast<long long>(v) * p.vtiles + blockIdx.x];
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    p.view_off[v] = static_cast<long long>(out);
    if (v == p.V - 1) p.view_off[p.V] = static_cast<long long>(*p.scan_total);
  }
  for (int it = 0; it < COMPACT_ITERS; ++it) {
    const long long o = base + it * COMPACT_THREADS + threadIdx.x;
    const bool keep[1] = {o < p.m && p.view[o] == v};
    unsigned int rank[1], sum[1];
    chunk_ranks<1>(keep, rank, sum);
    if (keep[0]) p.view_obs[out + rank[0]] = static_cast<int>(o);
    out += sum[0];
  }
}

// ------------------------------------------------------------------------------------------------------ cost and control
// grid tblocks.  trial = 0: the cost at the current parameters (once, before the first step).  trial = 1: the trial point
// x + delta (written to the other buffer), its cost, whether an included observation has Z <= 0, the model decrease
// sum w (-r^T J delta - |J delta|^2 / 2) = -g^T delta - delta^T H delta / 2 at the current linearisation, |delta_p|^2 and
// |P|^2.  Partials per block: cost, model, |delta_p|^2, |P|^2, behind count, included observations.
__global__ void __launch_bounds__(BA_THREADS, 1) ba_eval_kernel(const BaParams p, int trial) {
  __shared__ double red[BA_THREADS / 32];
  const BaState* s = p.st;
  if (s->stop || (trial && s->small)) return;
  const int cur = s->cur;
  const long long n3 = 3 * p.n;
  const double* cam = p.cam + (trial ? 1 - cur : cur) * p.V * BA_CAM;
  const long long t = static_cast<long long>(blockIdx.x) * BA_THREADS + threadIdx.x;
  double acc[BA_EVAL] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (t < p.n) {
    const double* P0 = p.pts + cur * n3 + 3 * t;
    const bool in = p.incl[t];
    double c[3] = {P0[0], P0[1], P0[2]}, d[3] = {0.0, 0.0, 0.0};
    if (in) {
      acc[3] = c[0] * c[0] + c[1] * c[1] + c[2] * c[2];
      if (trial) {
#pragma unroll
        for (int a = 0; a < 3; ++a) {
          d[a] = p.dp[3 * t + a];
          c[a] = c[a] + d[a];
        }
        acc[2] = d[0] * d[0] + d[1] * d[1] + d[2] * d[2];
      }
    }
    if (trial)
#pragma unroll
      for (int a = 0; a < 3; ++a) p.pts[(1 - cur) * n3 + 3 * t + a] = c[a];
    if (in) {
      long long b, e;
      ba_obs_range(p, t, b, e);
      for (long long q = b; q < e; ++q) {
        const int v = p.view[q];
        const double* C = cam + v * BA_CAM;
        double X[3], du, dv;
        acc[4] += track_reproject(C, C + 12, c, p.obs[2 * q], p.obs[2 * q + 1], X, du, dv) ? 1.0 : 0.0;
        acc[0] += 0.5 * ba_rho(p, du * du + dv * dv);
        acc[5] += 1.0;
        if (trial) {
          const BaObs& o = p.ob[q];
          const double* dc = p.dcam + v * BA_NP;
          double jd[2];
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            double a = 0.0;
#pragma unroll
            for (int i = 0; i < BA_NP; ++i) a += o.jc[r][i] * dc[i];
            jd[r] = a + (o.jp[r][0] * d[0] + o.jp[r][1] * d[1] + o.jp[r][2] * d[2]);
          }
          acc[1] += o.w * (-(o.r[0] * jd[0] + o.r[1] * jd[1]) - 0.5 * (jd[0] * jd[0] + jd[1] * jd[1]));
        }
      }
    }
  }
#pragma unroll
  for (int k = 0; k < BA_EVAL; ++k) {
    const double v = ba_block_sum<BA_THREADS>(acc[k], red);
    if (threadIdx.x == 0) p.epart[blockIdx.x * BA_EVAL + k] = v;
  }
}

// one block of BA_PCG_THREADS: the eval partials summed in a fixed order, then thread 0 decides.  init = 1 after the first
// evaluation: the initial cost, status 3 when no observation is refined.
__global__ void __launch_bounds__(BA_PCG_THREADS) ba_control_kernel(const BaParams p, int init) {
  __shared__ double red[BA_PCG_THREADS / 32];
  BaState* s = p.st;
  if (s->stop) return;
  double acc[BA_EVAL];
  const bool evaluated = init || !s->small;
  for (int k = 0; k < BA_EVAL; ++k) {
    double v = 0.0;
    if (evaluated)
      for (int b = threadIdx.x; b < p.tblocks; b += BA_PCG_THREADS) v += p.epart[b * BA_EVAL + k];
    acc[k] = ba_block_sum<BA_PCG_THREADS>(v, red);
  }
  if (threadIdx.x != 0) return;
  if (init) {
    s->cost = acc[0];
    p.cost_out[0] = acc[0];
    if (acc[5] == 0.0) {
      s->stop = 1;
      s->status = 3;
    }
  } else if (s->small) {
    s->stop = 1;
    s->status = 0;
  } else {
    s->steps += 1;
    s->pcg += s->its;
    const double step = sqrt(s->cam_step2 + acc[2]), xnorm = sqrt(s->cam_x2 + acc[3]);
    if (step <= 1e-8 * (xnorm + 1e-8)) {
      s->stop = 1;
      s->status = 0;
    } else {
      const double f = s->cost, fn = acc[0], model = acc[1];
      const double rho = (f - fn) / model;
      if (acc[4] == 0.0 && isfinite(fn) && model > 0.0 && rho > 1e-3) {
        const double q = 2.0 * rho - 1.0;
        s->mu = s->mu / fmax(1.0 / 3.0, 1.0 - q * q * q);
        s->nu = 2.0;
        s->cost = fn;
        s->cur ^= 1;
        s->accepted += 1;
        s->lin = 1;
        if (f - fn <= 1e-6 * f) {
          s->stop = 1;
          s->status = 0;
        }
      } else {
        s->mu = s->mu / s->nu;
        s->nu = 2.0 * s->nu;
        s->lin = 0;
        if (s->mu < 1e-32) {
          s->stop = 1;
          s->status = 2;
        }
      }
    }
    if (p.trace) p.trace[s->steps - 1] = s->cost;
    if (!s->stop && s->steps >= p.iterations) {
      s->stop = 1;
      s->status = 1;
    }
  }
  s->small = 0;
  s->arrive = 0u;
}

// ----------------------------------------------------------------------------------------------------------- linear system
// Residual and Jacobians of one observation at camera C (BA_CAM doubles), point c; mask m of the view's parameters.
__device__ __forceinline__ void ba_linearize(const BaParams& p, const double* C, const double* m, const double c[3], double ox,
                                             double oy, BaObs& o) {
  double X[3], du, dv;
  track_reproject(C, C + 12, c, ox, oy, X, du, dv);
  const double iz = 1.0 / X[2], xn = X[0] / X[2], yn = X[1] / X[2];
  const double a[3] = {X[0] - C[3], X[1] - C[7], X[2] - C[11]};      // R c
  const double fxz = C[12] * iz, fyz = C[16] * iz;
  const double jc[2][BA_NP] = {{fxz * (-xn * a[1]), fxz * (a[2] + xn * a[0]), fxz * (-a[1]), fxz, 0.0, -fxz * xn, xn, 0.0},
                               {fyz * (-a[2] - yn * a[1]), fyz * (yn * a[0]), fyz * a[0], 0.0, fyz, -fyz * yn, 0.0, yn}};
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int i = 0; i < BA_NP; ++i) o.jc[r][i] = m[i] != 0.0 ? jc[r][i] : 0.0;
#pragma unroll
  for (int b = 0; b < 3; ++b) {
    o.jp[0][b] = fxz * (C[b] - xn * C[8 + b]);
    o.jp[1][b] = fyz * (C[4 + b] - yn * C[8 + b]);
  }
  o.r[0] = du;
  o.r[1] = dv;
  o.w = ba_weight(p, du * du + dv * dv);
  o.pad = 0.0;
}

// per track: Jacobians at the current parameters after an accepted step (or the first), V_p and g_p from them,
// (V_p + D_p / mu)^-1 by cofactors, V_p^-1 g_p; block max of |g_p|
__global__ void __launch_bounds__(BA_THREADS) ba_track_kernel(const BaParams p) {
  __shared__ double red[BA_THREADS / 32];
  const BaState* s = p.st;
  if (s->stop) return;
  const int cur = s->cur, lin = s->lin;
  const double mu = s->mu;
  const long long t = static_cast<long long>(blockIdx.x) * BA_THREADS + threadIdx.x;
  double gm = 0.0;
  if (t < p.n) {
    long long b, e;
    ba_obs_range(p, t, b, e);
    const bool in = p.incl[t];
    const double* P = p.pts + cur * 3 * p.n + 3 * t;
    const double c[3] = {P[0], P[1], P[2]};
    double H[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, g[3] = {0.0, 0.0, 0.0};
    for (long long q = b; q < e; ++q) {
      BaObs& o = p.ob[q];
      if (lin) {
        if (in) {
          const int v = p.view[q];
          ba_linearize(p, p.cam + (cur * p.V + v) * BA_CAM, p.mask + v * BA_NP, c, p.obs[2 * q], p.obs[2 * q + 1], o);
        } else {
          double* z = reinterpret_cast<double*>(&o);
          for (int k = 0; k < BA_OBS_DOUBLES; ++k) z[k] = 0.0;
        }
      }
      if (!in) continue;
      const double w = o.w;
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const double* j = o.jp[r];
        H[0] += w * (j[0] * j[0]);
        H[1] += w * (j[1] * j[0]);
        H[2] += w * (j[1] * j[1]);
        H[3] += w * (j[2] * j[0]);
        H[4] += w * (j[2] * j[1]);
        H[5] += w * (j[2] * j[2]);
        g[0] += w * (j[0] * o.r[r]);
        g[1] += w * (j[1] * o.r[r]);
        g[2] += w * (j[2] * o.r[r]);
      }
    }
    double inv[9] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0}, y[3] = {0.0, 0.0, 0.0};
    if (in) {
      const double a = H[0] + ba_clamp(H[0]) / mu, d = H[2] + ba_clamp(H[2]) / mu, f = H[5] + ba_clamp(H[5]) / mu;
      const double bb = H[1], c2 = H[3], e2 = H[4];
      // symmetric [[a, bb, c2], [bb, d, e2], [c2, e2, f]]
      const double A = d * f - e2 * e2, B = c2 * e2 - bb * f, Cc = bb * e2 - c2 * d;
      const double det = a * A + bb * B + c2 * Cc;
      const double D = c2 * bb - a * e2, F = a * d - bb * bb, E = a * f - c2 * c2;
      inv[0] = A / det; inv[1] = B / det; inv[2] = Cc / det;
      inv[3] = B / det; inv[4] = E / det; inv[5] = D / det;
      inv[6] = Cc / det; inv[7] = D / det; inv[8] = F / det;
#pragma unroll
      for (int r = 0; r < 3; ++r) y[r] = inv[3 * r] * g[0] + inv[3 * r + 1] * g[1] + inv[3 * r + 2] * g[2];
      gm = fmax(fabs(g[0]), fmax(fabs(g[1]), fabs(g[2])));
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) p.vinv[9 * t + k] = inv[k];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      p.y[3 * t + k] = y[k];
      p.gp[3 * t + k] = g[k];
    }
  }
  gm = ba_block_max<BA_THREADS>(gm, red);
  if (threadIdx.x == 0) p.gmax[blockIdx.x] = gm;
}

// One per-view sum entry of one staged observation d (BA_STAGE doubles): e < 36 U_ij, e < 72 (W V^-1 W^T)_ij, e < 80 g_i,
// e < 88 (W V^-1 g_p)_i, with W_i = w (jc[0][i] jp[0] + jc[1][i] jp[1]).
__device__ __forceinline__ double ba_entry(const double* d, int e, int i, int j) {
  const double* jc0 = d;
  const double* jc1 = d + BA_NP;
  const double* jp0 = d + 16;
  const double* jp1 = d + 19;
  const double w = d[24];
  if (e < 36) return w * (jc0[i] * jc0[j] + jc1[i] * jc1[j]);
  double wi[3];
#pragma unroll
  for (int a = 0; a < 3; ++a) wi[a] = w * (jc0[i] * jp0[a] + jc1[i] * jp1[a]);
  if (e < 72) {
    const double* vi = d + 25;
    double wj[3], s = 0.0;
#pragma unroll
    for (int a = 0; a < 3; ++a) wj[a] = w * (jc0[j] * jp0[a] + jc1[j] * jp1[a]);
#pragma unroll
    for (int a = 0; a < 3; ++a) s += wi[a] * (vi[3 * a] * wj[0] + vi[3 * a + 1] * wj[1] + vi[3 * a + 2] * wj[2]);
    return s;
  }
  if (e < 80) return w * (jc0[i] * d[22] + jc1[i] * d[23]);
  return wi[0] * d[34] + wi[1] * d[35] + wi[2] * d[36];
}

__device__ __forceinline__ void ba_chunk(const BaParams& p, int v, int c, int chunks, long long& o0, long long& lo, long long& hi) {
  o0 = p.view_off[v];
  const long long nv = p.view_off[v + 1] - o0;
  const long long cs = (nv + chunks - 1) / chunks;
  lo = min(static_cast<long long>(c) * cs, nv);
  hi = min(lo + cs, nv);
}

// grid (BA_BLOCK_CHUNKS, V), BA_BLOCK_THREADS: thread e < BA_ENTRIES sums entry e over the chunk's observations in order
__global__ void __launch_bounds__(BA_BLOCK_THREADS) ba_view_block_kernel(const BaParams p) {
  __shared__ double sh[BA_BLOCK_BATCH][BA_STAGE];
  if (p.st->stop) return;
  const int v = blockIdx.y, e = threadIdx.x;
  long long o0, lo, hi;
  ba_chunk(p, v, blockIdx.x, BA_BLOCK_CHUNKS, o0, lo, hi);
  int i = 0, j = 0;
  if (e < 72) {
    const int k = e < 36 ? e : e - 36;
    while (ba_pk(i + 1, 0) <= k) ++i;
    j = k - ba_pk(i, 0);
  } else {
    i = (e - 72) & 7;
  }
  double acc = 0.0;
  for (long long base = lo; base < hi; base += BA_BLOCK_BATCH) {
    const int cnt = static_cast<int>(min(static_cast<long long>(BA_BLOCK_BATCH), hi - base));
    for (int idx = threadIdx.x; idx < cnt * BA_STAGE; idx += BA_BLOCK_THREADS) {
      const int k = idx / BA_STAGE, f = idx - k * BA_STAGE;
      const int o = p.view_obs[o0 + base + k];
      const long long t = p.obs_track[o];
      sh[k][f] = f < 25 ? reinterpret_cast<const double*>(p.ob + o)[f] : f < 34 ? p.vinv[9 * t + f - 25] : p.y[3 * t + f - 34];
    }
    __syncthreads();
    if (e < BA_ENTRIES)
      for (int k = 0; k < cnt; ++k) acc += ba_entry(sh[k], e, i, j);
    __syncthreads();
  }
  if (e < BA_ENTRIES) p.vpart[(static_cast<long long>(v) * BA_BLOCK_CHUNKS + blockIdx.x) * BA_ENTRIES + e] = acc;
}

// grid V, BA_BLOCK_THREADS: the chunk partials of view v summed in chunk order
__global__ void __launch_bounds__(BA_BLOCK_THREADS) ba_view_reduce_kernel(const BaParams p) {
  if (p.st->stop || threadIdx.x >= BA_ENTRIES) return;
  const double* part = p.vpart + static_cast<long long>(blockIdx.x) * BA_BLOCK_CHUNKS * BA_ENTRIES + threadIdx.x;
  double s = 0.0;
  for (int c = 0; c < BA_BLOCK_CHUNKS; ++c) s += part[c * BA_ENTRIES];
  p.vsum[blockIdx.x * BA_ENTRIES + threadIdx.x] = s;
}

// ------------------------------------------------------------------------------------------------------------------- PCG
__device__ __forceinline__ void ba_grid_sync(unsigned* arrive, unsigned& target) {
  __syncthreads();
  target += gridDim.x;
  if (threadIdx.x == 0) {
    __threadfence();
    fps_red_release(arrive, 1u);
    while (static_cast<int>(fps_ld_acquire(arrive) - target) < 0) {
    }
  }
  __syncthreads();
}

// z = (L L^T)^-1 r, L packed lower
__device__ __forceinline__ void ba_chol_solve(const double* L, const double* r, double* z) {
  double y[BA_NP];
#pragma unroll
  for (int i = 0; i < BA_NP; ++i) {
    double s = r[i];
#pragma unroll
    for (int k = 0; k < i; ++k) s -= L[ba_pk(i, k)] * y[k];
    y[i] = s / L[ba_pk(i, i)];
  }
#pragma unroll
  for (int i = BA_NP - 1; i >= 0; --i) {
    double s = y[i];
#pragma unroll
    for (int k = i + 1; k < BA_NP; ++k) s -= L[ba_pk(k, i)] * z[k];
    z[i] = s / L[ba_pk(i, i)];
  }
}

// sum over the track's observations of w Jp^T (Jc x_v), x per view in shared memory at stride BA_NP
__device__ __forceinline__ void ba_wt_x(const BaParams& p, long long t, const double* x, double s[3]) {
  long long b, e;
  ba_obs_range(p, t, b, e);
  s[0] = s[1] = s[2] = 0.0;
  for (long long q = b; q < e; ++q) {
    const BaObs& o = p.ob[q];
    const double* xv = x + p.view[q] * BA_NP;
    double a[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      double u = 0.0;
#pragma unroll
      for (int i = 0; i < BA_NP; ++i) u += o.jc[r][i] * xv[i];
      a[r] = o.w * u;
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) s[k] += o.jp[0][k] * a[0] + o.jp[1][k] * a[1];
  }
}

// Cooperative, grid from the occupancy query; dynamic shared memory BA_VIEW_SMEM doubles per view.  Each CTA holds every
// view's U* = U + D / mu, the Cholesky factor of S_vv and the PCG vectors, and repeats the per-view steps; the two passes of
// S p run over the grid and meet on an arrival counter (release / acquire, as fps_grid_kernel).
__global__ void __launch_bounds__(BA_PCG_THREADS) ba_pcg_kernel(const BaParams p) {
  extern __shared__ double sm[];
  __shared__ double red[BA_PCG_THREADS / 32];
  BaState* s = p.st;
  if (s->stop) return;
  const int V = p.V, v = threadIdx.x;
  const bool owner = v < V;
  const double mu = s->mu;
  const int cur = s->cur;
  // gradient test: |g|inf over the points (per-block maxima) and the cameras
  double gm = 0.0;
  for (int i = threadIdx.x; i < p.tblocks; i += BA_PCG_THREADS) gm = fmax(gm, p.gmax[i]);
  for (int i = threadIdx.x; i < V * BA_NP; i += BA_PCG_THREADS) gm = fmax(gm, fabs(p.vsum[(i / BA_NP) * BA_ENTRIES + 72 + i % BA_NP]));
  gm = ba_block_max<BA_PCG_THREADS>(gm, red);
  if (gm <= 1e-10) {
    if (blockIdx.x == 0 && threadIdx.x == 0) s->small = 1;
    return;
  }
  double* U = sm + v * BA_PACK;
  double* L = sm + V * BA_PACK + v * BA_PACK;
  double* x = sm + 72 * V;
  double* r = sm + 80 * V;
  double* pv = sm + 88 * V;
  double* q = sm + 96 * V;
  double rz_v = 0.0, bb_v = 0.0;
  if (owner) {
    const double* e = p.vsum + v * BA_ENTRIES;
    for (int k = 0; k < BA_PACK; ++k) U[k] = e[k];
#pragma unroll
    for (int i = 0; i < BA_NP; ++i) U[ba_pk(i, i)] += ba_clamp(e[ba_pk(i, i)]) / mu;
    for (int k = 0; k < BA_PACK; ++k) L[k] = U[k] - e[36 + k];
    for (int j = 0; j < BA_NP; ++j) {                        // Cholesky of S_vv in place
      double d = L[ba_pk(j, j)];
      for (int k = 0; k < j; ++k) d -= L[ba_pk(j, k)] * L[ba_pk(j, k)];
      d = sqrt(d);
      L[ba_pk(j, j)] = d;
      for (int i = j + 1; i < BA_NP; ++i) {
        double a = L[ba_pk(i, j)];
        for (int k = 0; k < j; ++k) a -= L[ba_pk(i, k)] * L[ba_pk(j, k)];
        L[ba_pk(i, j)] = a / d;
      }
    }
    double* xv = x + v * BA_NP;
    double* rv = r + v * BA_NP;
    double* pvv = pv + v * BA_NP;
    double z[BA_NP];
#pragma unroll
    for (int i = 0; i < BA_NP; ++i) {
      xv[i] = 0.0;
      rv[i] = -e[72 + i] + e[80 + i];
      bb_v += rv[i] * rv[i];
    }
    ba_chol_solve(L, rv, z);
#pragma unroll
    for (int i = 0; i < BA_NP; ++i) {
      pvv[i] = z[i];
      rz_v += rv[i] * z[i];
    }
  }
  double rz = ba_block_sum<BA_PCG_THREADS>(rz_v, red);
  const double bb = ba_block_sum<BA_PCG_THREADS>(bb_v, red);
  const double tol = 1e-10 * sqrt(bb);
  double rr = bb;
  int it = 0;
  unsigned target = 0u;
  const long long tid = static_cast<long long>(blockIdx.x) * BA_PCG_THREADS + threadIdx.x;
  const long long nthreads = static_cast<long long>(gridDim.x) * BA_PCG_THREADS;
  const int lane = threadIdx.x & 31;
  for (;;) {
    if (it >= BA_PCG_MAX || !(sqrt(rr) > tol)) break;
    __syncthreads();                                           // the owners' p (previous iteration) before pass 1 reads it
    // pass 1, per track: z_p = V_p^-1 sum W^T p_v
    for (long long t = tid; t < p.n; t += nthreads) {
      double zz[3] = {0.0, 0.0, 0.0};
      if (p.incl[t]) {
        double a[3];
        ba_wt_x(p, t, pv, a);
        const double* vi = p.vinv + 9 * t;
#pragma unroll
        for (int k = 0; k < 3; ++k) zz[k] = vi[3 * k] * a[0] + vi[3 * k + 1] * a[1] + vi[3 * k + 2] * a[2];
      }
#pragma unroll
      for (int k = 0; k < 3; ++k) p.zt[3 * t + k] = zz[k];
    }
    ba_grid_sync(&s->arrive, target);
    // pass 2, per view and chunk (one warp each): sum W z_p over the chunk
    for (long long item = tid >> 5; item < static_cast<long long>(V) * BA_PCG_CHUNKS; item += nthreads >> 5) {
      const int iv = static_cast<int>(item / BA_PCG_CHUNKS), ic = static_cast<int>(item % BA_PCG_CHUNKS);
      long long o0, lo, hi;
      ba_chunk(p, iv, ic, BA_PCG_CHUNKS, o0, lo, hi);
      double acc[BA_NP] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
#pragma unroll 1
      for (long long k = lo + lane; k < hi; k += 32) {
        const int o = p.view_obs[o0 + k];
        const long long t = p.obs_track[o];
        const BaObs& ob = p.ob[o];
        const double z0 = __ldcg(p.zt + 3 * t), z1 = __ldcg(p.zt + 3 * t + 1), z2 = __ldcg(p.zt + 3 * t + 2);
        const double a0 = ob.w * (ob.jp[0][0] * z0 + ob.jp[0][1] * z1 + ob.jp[0][2] * z2);
        const double a1 = ob.w * (ob.jp[1][0] * z0 + ob.jp[1][1] * z1 + ob.jp[1][2] * z2);
#pragma unroll
        for (int i = 0; i < BA_NP; ++i) acc[i] += ob.jc[0][i] * a0 + ob.jc[1][i] * a1;
      }
#pragma unroll
      for (int i = 0; i < BA_NP; ++i) {
        double a = acc[i];
        for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
        if (lane == 0) p.bpart[item * BA_NP + i] = a;
      }
    }
    ba_grid_sync(&s->arrive, target);
    // per view, in every CTA: q = U* p - sum W z, alpha, x, r
    double pq_v = 0.0;
    if (owner) {
      const double* pvv = pv + v * BA_NP;
      double* qv = q + v * BA_NP;
      const double* part = p.bpart + static_cast<long long>(v) * BA_PCG_CHUNKS * BA_NP;
#pragma unroll
      for (int i = 0; i < BA_NP; ++i) {
        double a = 0.0;
#pragma unroll
        for (int k = 0; k < BA_NP; ++k) a += U[i >= k ? ba_pk(i, k) : ba_pk(k, i)] * pvv[k];
        double w = 0.0;
        for (int c = 0; c < BA_PCG_CHUNKS; ++c) w += __ldcg(part + c * BA_NP + i);
        qv[i] = a - w;
        pq_v += pvv[i] * qv[i];
      }
    }
    const double pq = ba_block_sum<BA_PCG_THREADS>(pq_v, red);
    if (!(pq > 0.0)) break;
    const double alpha = rz / pq;
    double rr_v = 0.0;
    if (owner)
#pragma unroll
      for (int i = 0; i < BA_NP; ++i) {
        x[v * BA_NP + i] += alpha * pv[v * BA_NP + i];
        r[v * BA_NP + i] -= alpha * q[v * BA_NP + i];
        rr_v += r[v * BA_NP + i] * r[v * BA_NP + i];
      }
    rr = ba_block_sum<BA_PCG_THREADS>(rr_v, red);
    ++it;
    if (it >= BA_PCG_MAX || !(sqrt(rr) > tol)) break;
    double rz_n = 0.0;
    if (owner) {
      ba_chol_solve(L, r + v * BA_NP, q + v * BA_NP);
#pragma unroll
      for (int i = 0; i < BA_NP; ++i) rz_n += r[v * BA_NP + i] * q[v * BA_NP + i];
    }
    const double rzn = ba_block_sum<BA_PCG_THREADS>(rz_n, red);
    const double beta = rzn / rz;
    rz = rzn;
    if (owner)
#pragma unroll
      for (int i = 0; i < BA_NP; ++i) pv[v * BA_NP + i] = q[v * BA_NP + i] + beta * pv[v * BA_NP + i];
  }
  __syncthreads();
  // back-substitution: delta_p = V_p^-1 (-g_p - sum W^T dc)
  for (long long t = tid; t < p.n; t += nthreads) {
    double d[3] = {0.0, 0.0, 0.0};
    if (p.incl[t]) {
      double a[3];
      ba_wt_x(p, t, x, a);
      const double* vi = p.vinv + 9 * t;
      const double h[3] = {-p.gp[3 * t] - a[0], -p.gp[3 * t + 1] - a[1], -p.gp[3 * t + 2] - a[2]};
#pragma unroll
      for (int k = 0; k < 3; ++k) d[k] = vi[3 * k] * h[0] + vi[3 * k + 1] * h[1] + vi[3 * k + 2] * h[2];
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) p.dp[3 * t + k] = d[k];
  }
  if (blockIdx.x != 0) return;
  // CTA 0: the camera step, the trial cameras, the camera parts of |delta| and |x|
  double step_v = 0.0, x_v = 0.0;
  if (owner) {
    const double* m = p.mask + v * BA_NP;
    const double* C = p.cam + (cur * V + v) * BA_CAM;
    double* T = p.cam + ((1 - cur) * V + v) * BA_CAM;
    double dc[BA_NP];
#pragma unroll
    for (int i = 0; i < BA_NP; ++i) {
      dc[i] = m[i] != 0.0 ? x[v * BA_NP + i] : 0.0;
      p.dcam[v * BA_NP + i] = dc[i];
      step_v += dc[i] * dc[i];
    }
#pragma unroll
    for (int k = 0; k < BA_CAM; ++k) T[k] = C[k];
    if (m[0] != 0.0) {                                         // R <- Exp(w) R, Rodrigues, series form for tiny angles
      const double w0 = dc[0], w1 = dc[1], w2 = dc[2];
      const double th2 = w0 * w0 + w1 * w1 + w2 * w2;
      double A = 1.0, B = 0.5;
      if (th2 >= 1e-16) {
        const double th = sqrt(th2);
        A = sin(th) / th;
        B = (1.0 - cos(th)) / th2;
      }
      const double w[3] = {w0, w1, w2};
      const double K[3][3] = {{0.0, -w2, w1}, {w2, 0.0, -w0}, {-w1, w0, 0.0}};
      double Ex[3][3];
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) Ex[i][j] = (i == j ? 1.0 - B * th2 : 0.0) + B * (w[i] * w[j]) + A * K[i][j];
#pragma unroll
      for (int i = 0; i < 3; ++i)
#pragma unroll
        for (int j = 0; j < 3; ++j) T[4 * i + j] = Ex[i][0] * C[j] + Ex[i][1] * C[4 + j] + Ex[i][2] * C[8 + j];
    }
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      if (m[3 + a] != 0.0) {
        T[4 * a + 3] = C[4 * a + 3] + dc[3 + a];
        x_v += C[4 * a + 3] * C[4 * a + 3];
      }
    }
    if (m[6] != 0.0) {
      T[12] = C[12] + dc[6];
      x_v += C[12] * C[12];
    }
    if (m[7] != 0.0) {
      T[16] = C[16] + dc[7];
      x_v += C[16] * C[16];
    }
  }
  const double step2 = ba_block_sum<BA_PCG_THREADS>(step_v, red);
  const double x2 = ba_block_sum<BA_PCG_THREADS>(x_v, red);
  if (threadIdx.x == 0) {
    s->cam_step2 = step2;
    s->cam_x2 = x2;
    s->its = it;
  }
}

// ---------------------------------------------------------------------------------------------------------------- outputs
// per track: the refined point and its error, the formula and order of track_point_kernel
__global__ void __launch_bounds__(BA_THREADS) ba_output_kernel(const BaParams p) {
  const long long t = static_cast<long long>(blockIdx.x) * BA_THREADS + threadIdx.x;
  if (t >= p.n) return;
  const int cur = p.st->cur;
  const double* P = p.pts + cur * 3 * p.n + 3 * t;
  const double c[3] = {P[0], P[1], P[2]};
#pragma unroll
  for (int a = 0; a < 3; ++a) p.points_out[3 * t + a] = c[a];
  long long b, e;
  ba_obs_range(p, t, b, e);
  double err = 0.0;
  bool behind = false;
  for (long long q = b; q < e; ++q) {
    const double* C = p.cam + (cur * p.V + p.view[q]) * BA_CAM;
    double X[3], du, dv;
    behind |= track_reproject(C, C + 12, c, p.obs[2 * q], p.obs[2 * q + 1], X, du, dv);
    err = __dadd_rn(err, __dsqrt_rn(__dadd_rn(__dmul_rn(du, du), __dmul_rn(dv, dv))));
  }
  p.error_out[t] = behind ? __longlong_as_double(0x7ff0000000000000LL) : __ddiv_rn(err, static_cast<double>(e - b));
}

// one block of 32: cameras (K's other entries copied from the input), cost and counters
__global__ void ba_finish_kernel(const BaParams p) {
  const BaState* s = p.st;
  const double* cam = p.cam + s->cur * p.V * BA_CAM;
  for (int v = threadIdx.x; v < p.V; v += blockDim.x) {
#pragma unroll
    for (int i = 0; i < 12; ++i) p.ext_out[12 * v + i] = cam[v * BA_CAM + i];
#pragma unroll
    for (int i = 0; i < 9; ++i) p.intr_out[9 * v + i] = p.intr[9 * v + i];
    p.intr_out[9 * v] = cam[v * BA_CAM + 12];
    p.intr_out[9 * v + 4] = cam[v * BA_CAM + 16];
  }
  if (threadIdx.x == 0) {
    p.cost_out[1] = s->cost;
    p.stats_out[0] = s->steps;
    p.stats_out[1] = s->accepted;
    p.stats_out[2] = s->pcg;
    p.stats_out[3] = s->status;
  }
}

}  // namespace ovg
