/* A host written in C drives the hot path through the handle-level C ABI (include/ovg.h, "Runtime") with raw device pointers:
 * no Python, no torch.  Property checked: with all-zero block weights every block is the identity, so the kept
 * intermediates must equal the assembled tokens (camera / register / patch + depth placeholder; reference
 * omnivggt_aggregator.py:155-156,:202-213,:248-251) rounded to bf16, and cam_out the camera token rows in fp32.
 *
 *   gcc runtime_identity.c -I include -L <pkg> -lovg -L /usr/local/cuda/lib64 -lcudart -lm -o runtime_identity
 */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "ovg.h"

/* minimal CUDA runtime prototypes (libcudart), so that the test needs no CUDA headers */
typedef int cudaError_t;
cudaError_t cudaMalloc(void** p, size_t n);
cudaError_t cudaMemset(void* p, int v, size_t n);
cudaError_t cudaMemcpy(void* dst, const void* src, size_t n, int kind);
cudaError_t cudaDeviceSynchronize(void);
const char* cudaGetErrorString(cudaError_t e);
enum { H2D = 1, D2H = 2 };

#define CK(x) do { cudaError_t e_ = (x); if (e_) { printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); return 2; } } while (0)
#define OK(x) do { int r_ = (x); if (r_) { printf("libovg error %d: %s (%s:%d)\n", r_, ovg_last_error(), __FILE__, __LINE__); return 3; } } while (0)

static void* dzero(size_t bytes) {
  void* p = NULL;
  if (cudaMalloc(&p, bytes) || cudaMemset(p, 0, bytes)) return NULL;
  return p;
}
static void* dcopy(const void* h, size_t bytes) {
  void* p = NULL;
  if (cudaMalloc(&p, bytes) || cudaMemcpy(p, h, bytes, H2D)) return NULL;
  return p;
}
static float bf16_to_f32(uint16_t v) { uint32_t u = (uint32_t)v << 16; float f; memcpy(&f, &u, 4); return f; }
static float round_bf16(float f) {          /* round to nearest even, as __float2bfloat16 */
  uint32_t u; memcpy(&u, &f, 4);
  u += 0x7fffu + ((u >> 16) & 1u);
  u &= 0xffff0000u;
  memcpy(&f, &u, 4);
  return f;
}

int main(void) {
  enum { C = 128, R = 4, PATCH = 14, H = 28, W = 28, B = 1, S = 2, K = B * S, P = (H / PATCH) * (W / PATCH), T = P + R + 1 };
  OK(ovg_device_check());
  /* ---- weights: every matrix / bias / gamma zero (identity blocks); LayerNorm weights are irrelevant then */
  ovg_block_weights blk;
  memset(&blk, 0, sizeof blk);
  blk.ln1_w = dzero(C * 4); blk.ln1_b = dzero(C * 4); blk.ln2_w = dzero(C * 4); blk.ln2_b = dzero(C * 4);
  blk.w_qkv = dzero(3 * C * C * 2); blk.b_qkv = dzero(3 * C * 4);
  blk.qn_w = dzero(64 * 4); blk.qn_b = dzero(64 * 4); blk.kn_w = dzero(64 * 4); blk.kn_b = dzero(64 * 4);
  blk.w_proj = dzero(C * C * 2); blk.b_proj = dzero(C * 4); blk.g1 = dzero(C * 4);
  blk.w_fc1 = dzero(4 * C * C * 2); blk.b_fc1 = dzero(4 * C * 4); blk.w_fc2 = dzero(4 * C * C * 2); blk.b_fc2 = dzero(C * 4);
  blk.g2 = dzero(C * 4);
  float h_cam[2 * C], h_reg[2 * R * C], h_ph[C], h_ones[C];
  static float h_patch[K * P * C];
  for (int i = 0; i < 2 * C; ++i) h_cam[i] = 0.01f * (float)(i % 37) - 0.1f;
  for (int i = 0; i < 2 * R * C; ++i) h_reg[i] = 0.003f * (float)(i % 101) - 0.15f;
  for (int i = 0; i < C; ++i) { h_ph[i] = 0.5f - 0.004f * (float)i; h_ones[i] = 1.0f; }
  for (int i = 0; i < K * P * C; ++i) h_patch[i] = sinf(0.37f * (float)i);
  ovg_aggregator_desc d;
  memset(&d, 0, sizeof d);
  d.C = C; d.registers = R; d.depth = 1; d.patch = PATCH;
  d.frame_blocks = &blk; d.global_blocks = &blk;
  d.cam_tok = dcopy(h_cam, sizeof h_cam); d.reg_tok = dcopy(h_reg, sizeof h_reg); d.placeholder = dcopy(h_ph, sizeof h_ph);
  d.depth_w = dzero(C * 2 * PATCH * PATCH * 2); d.depth_b = dzero(C * 4); d.ones_c = dcopy(h_ones, sizeof h_ones);
  d.keep_layers[0] = d.keep_layers[1] = d.keep_layers[2] = d.keep_layers[3] = 0;
  ovg_aggregator* agg = NULL;
  OK(ovg_aggregator_create(&d, &agg));

  /* ---- inputs */
  float* patch = dcopy(h_patch, sizeof h_patch);
  float* inj = dzero((size_t)2 * K * C * 4);            /* [depth + 1, K, C] camera injection vectors: none */
  float h_cos[3 * 16], h_sin[3 * 16];                   /* rope tables for 3 positions (q = k = 0 anyway) */
  for (int i = 0; i < 48; ++i) { h_cos[i] = 1.0f; h_sin[i] = 0.0f; }
  float* cosd = dcopy(h_cos, sizeof h_cos);
  float* sind = dcopy(h_sin, sizeof h_sin);
  const long long wsb = ovg_aggregator_workspace_bytes(agg, B, S, H, W, 0);
  if (wsb <= 0) { printf("workspace query failed\n"); return 4; }
  void* ws = dzero((size_t)wsb);
  void* slots[4];
  for (int i = 0; i < 4; ++i) slots[i] = dzero((size_t)K * T * 2 * C * 2);
  float* cam_out = dzero((size_t)K * 2 * C * 4);
  if (!patch || !inj || !ws || !cam_out || !slots[3]) { printf("allocation failed\n"); return 5; }
  OK(ovg_aggregator_forward(agg, NULL, patch, inj, NULL, NULL, NULL, 0, NULL, 0, cosd, sind, 3, B, S, H, W, ws, wsb, slots, cam_out,
                            NULL, NULL));
  CK(cudaDeviceSynchronize());

  /* ---- check */
  static uint16_t h_slot[K * T * 2 * C];
  static float h_co[K * 2 * C];
  CK(cudaMemcpy(h_slot, slots[3], sizeof h_slot, D2H));
  CK(cudaMemcpy(h_co, cam_out, sizeof h_co, D2H));
  int bad = 0;
  for (int k = 0; k < K; ++k) {
    const int s = (k % S) == 0 ? 0 : 1;                 /* view 0 uses slot 0 of the camera / register tokens */
    for (int t = 0; t < T; ++t)
      for (int c = 0; c < C; ++c) {
        float x;
        if (t == 0) x = h_cam[s * C + c];
        else if (t <= R) x = h_reg[(s * R + (t - 1)) * C + c];
        else x = h_patch[(k * P + (t - 1 - R)) * C + c] + h_ph[c];
        const float want = round_bf16(x);
        const float f = bf16_to_f32(h_slot[((size_t)k * T + t) * 2 * C + c]);
        const float g = bf16_to_f32(h_slot[((size_t)k * T + t) * 2 * C + C + c]);
        if (f != want || g != want) { if (bad < 5) printf("slot mismatch k=%d t=%d c=%d: %g %g want %g\n", k, t, c, f, g, want); ++bad; }
        if (t == 0 && (h_co[k * 2 * C + c] != x || h_co[k * 2 * C + C + c] != x)) {
          if (bad < 5) printf("cam_out mismatch k=%d c=%d: %g %g want %g\n", k, c, h_co[k * 2 * C + c], h_co[k * 2 * C + C + c], x);
          ++bad;
        }
      }
  }
  ovg_aggregator_destroy(agg);
  printf("runtime_identity: %d mismatches, %lld libovg launches\n", bad, ovg_launch_count());
  return bad ? 1 : 0;
}
