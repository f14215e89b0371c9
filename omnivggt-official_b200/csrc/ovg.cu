// libovg C ABI (include/ovg.h): argument validation, TMA descriptor cache, kernel launches.
#include <atomic>
#include <cstdlib>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include <cudaTypedefs.h>

#include "../../include/ovg.h"
#include "attn.cuh"
#include "camera.cuh"
#include "elem.cuh"
#include "gemm.cuh"
#include "post.cuh"
#include "match.cuh"
#include "mesh.cuh"
#include "sky.cuh"
#include "fps.cuh"
#include "rank.cuh"
#include "tail.cuh"
#include "pre.cuh"
#include "jpeg.cuh"

namespace {

thread_local std::string g_err;
std::atomic<long long> g_launches{0};

int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

#define OVG_REQUIRE(cond, msg)                                                           \
  do {                                                                                   \
    if (!(cond)) return fail(OVG_E_INVALID, std::string(__func__) + ": " + (msg));        \
  } while (0)

#define OVG_CUDA(expr)                                                                   \
  do {                                                                                   \
    cudaError_t e__ = (expr);                                                            \
    if (e__ != cudaSuccess)                                                              \
      return fail(OVG_E_CUDA, std::string(__func__) + ": " #expr ": " + cudaGetErrorString(e__)); \
  } while (0)

int post_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(OVG_E_CUDA, std::string(what) + ": launch failed: " + cudaGetErrorString(e));
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return OVG_OK;
}

// ------------------------------------------------------------------------------ tensor maps
PFN_cuTensorMapEncodeTiled_v12000 get_encode() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess) p = nullptr;
    return reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }();
  return fn;
}

struct MapKey {
  const void* ptr;
  unsigned long long d0, d1, d2, ld, box1;   // box1 also carries (kind << 32) for output maps
  bool operator==(const MapKey& o) const {
    return ptr == o.ptr && d0 == o.d0 && d1 == o.d1 && d2 == o.d2 && ld == o.ld && box1 == o.box1;
  }
};
struct MapKeyHash {
  size_t operator()(const MapKey& k) const {
    size_t h = std::hash<const void*>()(k.ptr);
    for (unsigned long long v : {k.d0, k.d1, k.d2, k.ld, k.box1}) h = h * 1000003u ^ std::hash<unsigned long long>()(v);
    return h;
  }
};
std::mutex g_map_mu;
std::unordered_map<MapKey, CUtensorMap, MapKeyHash> g_maps;

// bf16 tensor [d2][d1][d0] (d0 contiguous, row stride ld elements, d2 stride d1*ld), box = [64, box1, 1], 128B swizzle.
// d2 == 0 -> rank 2.
int get_map(const void* ptr, unsigned long long d0, unsigned long long d1, unsigned long long d2,
            unsigned long long ld, unsigned box1, CUtensorMap* out) {
  MapKey key{ptr, d0, d1, d2, ld, box1};
  {
    std::lock_guard<std::mutex> g(g_map_mu);
    auto it = g_maps.find(key);
    if (it != g_maps.end()) {
      *out = it->second;
      return OVG_OK;
    }
  }
  auto enc = get_encode();
  if (!enc) return fail(OVG_E_CUDA, "cuTensorMapEncodeTiled entry point not available");
  if ((reinterpret_cast<uintptr_t>(ptr) & 15) || ((ld * 2) & 15))
    return fail(OVG_E_INVALID, "TMA operand must be 16-byte aligned with a 16-byte multiple row stride");
  cuuint64_t gdim[3] = {d0, d1, d2 ? d2 : 1};
  cuuint64_t gstr[2] = {ld * 2, d1 * ld * 2};
  cuuint32_t box[3] = {64, box1, 1};
  cuuint32_t estr[3] = {1, 1, 1};
  CUtensorMap m;
  CUresult r = enc(&m, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, d2 ? 3 : 2, const_cast<void*>(ptr), gdim, gstr, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(OVG_E_CUDA, "cuTensorMapEncodeTiled failed (" + std::to_string(int(r)) + ")");
  {
    std::lock_guard<std::mutex> g(g_map_mu);
    if (g_maps.size() > 8192) g_maps.clear();
    g_maps.emplace(key, m);
  }
  *out = m;
  return OVG_OK;
}

// Function attributes and the SM count are per device: one process may drive several GPUs (or several host threads).
constexpr int kMaxDevices = 64;
int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return dev >= 0 && dev < kMaxDevices ? dev : 0;
}
int num_sms() {
  static std::atomic<int> n[kMaxDevices];
  const int dev = current_device();
  int v = n[dev].load(std::memory_order_relaxed);
  if (v == 0) {
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    n[dev].store(v, std::memory_order_relaxed);
  }
  return v;
}
// true exactly until `mark_done` has been called for (slot, current device); setting an attribute twice is harmless
struct PerDeviceOnce {
  std::atomic<bool> done[kMaxDevices];
  bool needed() { return !done[current_device()].load(std::memory_order_acquire); }
  void mark_done() { done[current_device()].store(true, std::memory_order_release); }
};

// Lets Kernel launch with `bytes` of dynamic shared memory (more than the 48 KB default); set once per device.
template <auto Kernel>
int allow_dynamic_smem(int bytes) {
  static PerDeviceOnce once;
  if (once.needed()) {
    OVG_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
    once.mark_done();
  }
  return OVG_OK;
}

template <int BN, int EPI>
int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const ovg::GemmParams& p, cudaStream_t st) {
  using Cfg = ovg::GemmCfg<BN>;
  const int rc = allow_dynamic_smem<ovg::gemm_kernel<BN, EPI>>(Cfg::SMEM_BYTES);
  if (rc) return rc;
  const int tiles = ((p.M + 127) / 128) * ((p.N + BN - 1) / BN);
  const int grid = tiles < num_sms() ? tiles : num_sms();
  ovg::gemm_kernel<BN, EPI><<<grid, ovg::GEMM_THREADS, Cfg::SMEM_BYTES, st>>>(ta, tb, p);
  return post_launch("ovg_gemm");
}

template <int EPI>
int dispatch_bn(int bn, const CUtensorMap& ta, const CUtensorMap& tb, const ovg::GemmParams& p, cudaStream_t st) {
  switch (bn) {
    case 128: return launch_gemm<128, EPI>(ta, tb, p, st);
    case 64: return launch_gemm<64, EPI>(ta, tb, p, st);
    case 32: return launch_gemm<32, EPI>(ta, tb, p, st);
    default: return fail(OVG_E_INVALID, "ovg_gemm: unsupported block_n");
  }
}

}  // namespace

extern "C" {

int ovg_version(void) { return 4; }
const char* ovg_last_error(void) { return g_err.c_str(); }
long long ovg_launch_count(void) { return g_launches.load(); }

int ovg_device_check(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return fail(OVG_E_NODEVICE, "no CUDA device");
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) return fail(OVG_E_NODEVICE, "cannot query device");
  if (prop.major != 9 || prop.minor != 0)
    return fail(OVG_E_NODEVICE, std::string("libovg requires sm_90 (H100); found sm_") + std::to_string(prop.major) +
                                    std::to_string(prop.minor));
  return OVG_OK;
}

int ovg_gemm(const ovg_gemm_args* a, void* stream) {
  OVG_REQUIRE(a && a->a && a->b, "null operand");
  OVG_REQUIRE(a->m > 0 && a->n > 0 && a->a_cols > 0 && a->a_rows > 0, "empty problem");
  OVG_REQUIRE(a->num_taps >= 1 && a->num_taps <= 9, "num_taps must be in [1,9]");
  OVG_REQUIRE(a->a_cols % 8 == 0, "a_cols must be a multiple of 8");
  OVG_REQUIRE(a->num_taps == 1 || a->a_cols % 64 == 0, "multi-tap GEMM needs a_cols % 64 == 0");
  OVG_REQUIRE(a->n % 32 == 0, "n must be a multiple of 32");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);

  ovg::GemmParams p{};
  p.M = a->m;
  p.N = a->n;
  p.kc_blocks = (a->a_cols + 63) / 64;
  p.k_blocks = p.kc_blocks * a->num_taps;
  for (int i = 0; i < 9; ++i) p.tap_off[i] = i < a->num_taps ? a->tap_off[i] : 0;
  p.bias = a->bias;
  p.act = a->act;
  p.out = a->out;
  p.ldo = a->ldo;
  p.table = a->table;
  p.table_rows = a->table_rows > 0 ? a->table_rows : 1;
  p.f16 = (a->f16 && (a->epi == OVG_EPI_BF16 || a->epi == OVG_EPI_HEADTAIL)) ? 1 : 0;
  p.skip1 = reinterpret_cast<const __nv_bfloat16*>(a->skip1);
  p.skip2 = reinterpret_cast<const __nv_bfloat16*>(a->skip2);
  p.rowmap = a->rowmap;
  p.gh = a->gh;
  p.gw = a->gw;
  p.ps = a->ps;
  p.cout = a->cout;
  p.gamma = a->gamma;
  p.row_index = a->row_index;
  p.q_out = reinterpret_cast<__nv_bfloat16*>(a->q_out);
  p.k_out = reinterpret_cast<__nv_bfloat16*>(a->k_out);
  p.v_out = reinterpret_cast<__nv_bfloat16*>(a->v_out);
  p.C = a->C;
  p.ntok = a->ntok;
  p.T = a->T;
  p.nspecial = a->nspecial;
  p.wp = a->wp;
  p.maxpos = a->maxpos;
  p.qn_w = a->qn_w;
  p.qn_b = a->qn_b;
  p.kn_w = a->kn_w;
  p.kn_b = a->kn_b;
  p.rope_cos = a->rope_cos;
  p.rope_sin = a->rope_sin;
  p.qscale = a->qscale;
  p.qk_norm = a->qk_norm;
  p.rope = a->rope;
  p.w2 = a->w2;
  p.b2 = a->b2;
  p.outc = a->outc;
  p.head_act = a->head_act;
  p.preds = a->preds;
  p.conf = a->conf;
  p.n_peers = a->epi == OVG_EPI_QKV ? a->n_peers : 0;
  p.peer_ntok = a->peer_ntok;
  p.peer_tok_off = a->peer_tok_off;
  OVG_REQUIRE(p.n_peers >= 0 && p.n_peers <= 8, "at most 8 peers");
  for (int i = 0; i < p.n_peers; ++i) {
    OVG_REQUIRE(a->k_peers[i] && a->v_peers[i], "null peer buffer");
    p.k_peer[i] = reinterpret_cast<__nv_bfloat16*>(a->k_peers[i]);
    p.v_peer[i] = reinterpret_cast<__nv_bfloat16*>(a->v_peers[i]);
  }
  if (p.n_peers > 0) OVG_REQUIRE(a->peer_ntok >= a->ntok && a->peer_tok_off >= 0 && a->peer_tok_off + a->ntok <= a->peer_ntok,
                                 "peer token window");

  // block_n: 0 picks the tile width; any request above 128 (the widest tile on sm_90) runs as 128.
  int bn = a->block_n > 128 ? 128 : a->block_n;
  if (a->epi == OVG_EPI_HEADTAIL) {
    OVG_REQUIRE(a->n == 32, "HEADTAIL epilogue needs n == 32");
    OVG_REQUIRE(a->w2 && a->b2 && a->bias && a->preds && a->conf && a->outc >= 2 && a->outc <= 4, "HEADTAIL args");
    OVG_REQUIRE(a->rowmap == OVG_ROWS_PAD, "HEADTAIL runs on the zero-bordered grid");
    bn = 32;
  } else if (bn == 0) {
    bn = a->n >= 128 ? 128 : 64;
  }
  OVG_REQUIRE(bn == 32 || bn == 64 || bn == 128, "block_n must be 0, 32, 64 or >= 128");
  if (a->epi == OVG_EPI_QKV) {
    OVG_REQUIRE(a->q_out && a->bias && ((a->k_out && a->v_out) || a->n_peers > 0), "QKV args");
    if (a->qk_norm) OVG_REQUIRE(a->qn_w && a->qn_b && a->kn_w && a->kn_b, "QKV q/k norm weights");
    if (a->rope) OVG_REQUIRE(a->rope_cos && a->rope_sin && a->maxpos > 0 && a->maxpos <= 64 && a->wp > 0,
                             "QKV rope table (maxpos <= 64)");
    else p.maxpos = 0;
    OVG_REQUIRE(a->C % 64 == 0 && a->n == 3 * a->C && a->ntok > 0 && a->T > 0, "QKV geometry");
    if (p.wp <= 0) p.wp = 1;
    OVG_REQUIRE(a->m % a->ntok == 0, "m must be a multiple of ntok");
    if (bn < 64) bn = 64;
  } else if (a->epi == OVG_EPI_RESID) {
    OVG_REQUIRE(a->out && a->gamma && a->bias, "RESID needs out, gamma, bias");
  } else if (a->epi == OVG_EPI_BF16) {
    OVG_REQUIRE(a->out, "BF16 epilogue needs out");
    OVG_REQUIRE((reinterpret_cast<uintptr_t>(a->bias) & 15) == 0 && (reinterpret_cast<uintptr_t>(a->table) & 15) == 0 &&
                    (a->table == nullptr || a->n % 4 == 0),
                "bias / table must be 16-byte aligned");
    if (a->rowmap == OVG_ROWS_PIXSHUF)
      OVG_REQUIRE(a->ps > 0 && a->cout % 32 == 0 && a->n == a->ps * a->ps * a->cout, "PIXSHUF geometry");
    if (a->rowmap != OVG_ROWS_IDENT) OVG_REQUIRE(a->gh > 0 && a->gw > 0, "row map needs gh, gw");
  }

  CUtensorMap ta, tb;
  int rc = get_map(a->a, a->a_cols, a->a_rows, 0, a->lda, 128, &ta);
  if (rc) return rc;
  const unsigned long long ktot = static_cast<unsigned long long>(a->a_cols) * a->num_taps;
  rc = get_map(a->b, ktot, a->n, 0, a->ldb, bn, &tb);
  if (rc) return rc;

  switch (a->epi) {
    case OVG_EPI_BF16: return dispatch_bn<ovg::EPI_BF16>(bn, ta, tb, p, st);
    case OVG_EPI_RESID: return dispatch_bn<ovg::EPI_RESID>(bn, ta, tb, p, st);
    case OVG_EPI_QKV: return dispatch_bn<ovg::EPI_QKV>(bn, ta, tb, p, st);
    case OVG_EPI_HEADTAIL: {
      // row-shift kernel: 3x3 taps in row-major order over a 128-channel map ((ky, kx) -> tap_off = (ky-1)*pitch + kx-1)
      bool shape_ok = a->num_taps == 9 && a->a_cols == 128 && a->n == 32;
      for (int ky = 0; ky < 3 && shape_ok; ++ky)
        shape_ok = a->tap_off[ky * 3 + 1] - a->tap_off[ky * 3] == 1 && a->tap_off[ky * 3 + 2] - a->tap_off[ky * 3 + 1] == 1;
      if (!shape_ok) return launch_gemm<32, ovg::EPI_HEADTAIL>(ta, tb, p, st);
      CUtensorMap ta136;
      rc = get_map(a->a, a->a_cols, a->a_rows, 0, a->lda, ovg::HT_A_ROWS, &ta136);
      if (rc) return rc;
      rc = allow_dynamic_smem<ovg::headtail_kernel>(ovg::HT_SMEM_BYTES);
      if (rc) return rc;
      const int tiles = (p.M + ovg::GEMM_BM - 1) / ovg::GEMM_BM;
      const int grid = tiles < num_sms() ? tiles : num_sms();
      ovg::headtail_kernel<<<grid, ovg::HT_THREADS, ovg::HT_SMEM_BYTES, st>>>(ta136, tb, p);
      return post_launch("ovg_gemm(headtail)");
    }
    default: return fail(OVG_E_INVALID, "ovg_gemm: unknown epilogue");
  }
}

long long ovg_attention_scratch_bytes(void) { return 4LL * num_sms() * 128 * (64 * 4 + 8) + 256; }   // <= 4 parts of < one wave of tiles

int ovg_attention(const void* q, const void* k, const void* v, void* out, int batch, int heads, int nq, int nkv,
                  void* scratch, long long scratch_bytes, void* stream) {
  OVG_REQUIRE(q && k && v && out, "null operand");
  OVG_REQUIRE(batch > 0 && heads > 0 && nq > 0 && nkv > 0, "empty problem");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CUtensorMap tq, tk, tv;
  const unsigned long long bh = static_cast<unsigned long long>(batch) * heads;
  int rc = get_map(q, 64, nq, bh, 64, 128, &tq);
  if (rc) return rc;
  rc = get_map(k, 64, nkv, bh, 64, 128, &tk);
  if (rc) return rc;
  rc = get_map(v, 64, nkv, bh, 64, 128, &tv);
  if (rc) return rc;
  rc = allow_dynamic_smem<ovg::attn1_kernel>(ovg::ATT1_SMEM_BYTES);
  if (rc) return rc;
  const int q_tiles = (nq + 127) / 128;
  const long long tiles = static_cast<long long>(q_tiles) * heads * batch;
  OVG_REQUIRE(tiles < (1LL << 28), "too many tiles");
  ovg::AttnParams p{nq, nkv, heads, heads * 64, reinterpret_cast<__nv_bfloat16*>(out), q_tiles, static_cast<int>(tiles),
                    static_cast<int>(tiles), 1, nullptr, nullptr};
  // Short sequences (frame / DINOv2 attention: 11 KV tiles per item): one resident CTA per SM walks the items, so barrier
  // set-up is paid once and the next item's Q, K, V stream in under the current item's tail.  Long sequences keep one CTA
  // per item: the hardware's dynamic CTA placement balances the partial waves of the global attention.
  const int resident = num_sms();
  const int kv_tiles = (nkv + 127) / 128;
  const bool persistent = tiles > resident && kv_tiles <= 16;
  // Long sequences: the tiles of the last, partly empty wave are cut into 2-4 KV ranges (one CTA each, issued after the whole
  // tiles) whose partial (O, reference, row sum) a small kernel merges.
  int parts = 1;
  const int tail = static_cast<int>(tiles % resident);
  if (!persistent && scratch && tiles > resident && tail > 0 && kv_tiles >= 24) {
    double best = 1.0;
    for (int c = 2; c <= 4; ++c) {
      const double cost = static_cast<double>((static_cast<long long>(tail) * c + resident - 1) / resident) / c + 0.04;   // + merge
      if (cost < best - 0.1) {
        best = cost;
        parts = c;
      }
    }
    if (parts > 1) {
      const long long need = static_cast<long long>(tail) * parts * 128 * (64 * 4 + 8);
      if (need > scratch_bytes - 256 || (reinterpret_cast<uintptr_t>(scratch) & 15)) parts = 1;
    }
  }
  if (parts > 1) {
    p.n_full = static_cast<int>(tiles) - tail;
    p.parts = parts;
    p.items = p.n_full + tail * parts;
    p.part_o = static_cast<float*>(scratch);
    p.part_ml = reinterpret_cast<float2*>(p.part_o + static_cast<long long>(tail) * parts * 128 * 64);
  }
  const int grid1 = persistent ? resident : p.items;
  ovg::attn1_kernel<<<grid1, ovg::ATT1_THREADS, ovg::ATT1_SMEM_BYTES, st>>>(tq, tk, tv, p);
  rc = post_launch("ovg_attention");
  if (rc || parts <= 1) return rc;
  ovg::attn_merge_kernel<<<tail, 128, 0, st>>>(p);
  return post_launch("ovg_attention(merge)");
}

// in_mode: ovg::LN_IN_F32, LN_IN_BF16 or LN_IN_F32_AS_BF16 (the last is internal: ovg_dpt_forward_f32 reads fp32 layers with it)
static int layernorm(const void* in, int in_mode, long long ld_in, void* out, int out_is_f32, long long ld_out, int rows, int C,
                     const float* w, const float* b, float eps, int grp_out, int grp_in, int grp_off, void* stream) {
  OVG_REQUIRE(in && out && rows > 0, "null operand");
  OVG_REQUIRE(out_is_f32 >= 0 && out_is_f32 <= 2, "output type: 0 bf16, 1 fp32, 2 fp16");
  OVG_REQUIRE((w == nullptr) == (b == nullptr), "affine needs both weight and bias");
  OVG_REQUIRE(C % 128 == 0 && C <= 2048, "C must be a multiple of 128, <= 2048");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ovg::LnParams p{in, in_mode, ld_in, out, out_is_f32, ld_out, rows, C, w, b, eps,
                  grp_out, grp_in, grp_off};
  constexpr int ln_threads = 256;     // 8 rows per block
  constexpr int ln_persist = 2;       // persistent grid: blocks per SM
  OVG_REQUIRE((reinterpret_cast<uintptr_t>(w) & 15) == 0 && (reinterpret_cast<uintptr_t>(b) & 15) == 0, "w / b must be 16-byte aligned");
  const int rpb = ln_threads / 32;
  int blocks = (rows + rpb - 1) / rpb;
  if (blocks > num_sms() * ln_persist) blocks = num_sms() * ln_persist;
  switch (C / 32) {
#define OVG_LN_CASE(V) \
  case V: ovg::layernorm_kernel<V><<<blocks, ln_threads, 0, st>>>(p); break;
    OVG_LN_CASE(4) OVG_LN_CASE(8) OVG_LN_CASE(12) OVG_LN_CASE(16) OVG_LN_CASE(20) OVG_LN_CASE(24) OVG_LN_CASE(28)
    OVG_LN_CASE(32) OVG_LN_CASE(36) OVG_LN_CASE(40) OVG_LN_CASE(44) OVG_LN_CASE(48) OVG_LN_CASE(52) OVG_LN_CASE(56)
    OVG_LN_CASE(60) OVG_LN_CASE(64)
#undef OVG_LN_CASE
    default: return fail(OVG_E_INVALID, "ovg_layernorm: unsupported C");
  }
  return post_launch("ovg_layernorm");
}

int ovg_layernorm(const void* in, int in_is_bf16, long long ld_in, void* out, int out_is_f32, long long ld_out, int rows,
                  int C, const float* w, const float* b, float eps, int grp_out, int grp_in, int grp_off, void* stream) {
  return layernorm(in, in_is_bf16 ? ovg::LN_IN_BF16 : ovg::LN_IN_F32, ld_in, out, out_is_f32, ld_out, rows, C, w, b, eps, grp_out,
                   grp_in, grp_off, stream);
}

int ovg_assemble_tokens(float* x, const float* patch, const float* cam_tok, const float* reg_tok, const float* inj0,
                        const float* placeholder, const int* has_depth, int K, int S, int T, int R, int C, int view_base,
                        void* stream) {
  OVG_REQUIRE(x && patch && cam_tok && reg_tok && inj0 && placeholder && has_depth, "null operand");
  OVG_REQUIRE(K > 0 && S > 0 && K % S == 0 && T > R + 1 && C % 4 == 0, "bad geometry");
  ovg::AssembleParams p{x, patch, cam_tok, reg_tok, inj0, placeholder, has_depth, K, S, T, R, C, view_base};
  const int threads = C / 4 < 256 ? ((C / 4 + 31) / 32) * 32 : 256;
  ovg::assemble_tokens_kernel<<<K * T, threads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return post_launch("ovg_assemble_tokens");
}

int ovg_peer_barrier(int* const* flag_peers, int* epoch_counter, int rank, int world, void* stream) {
  OVG_REQUIRE(flag_peers && epoch_counter && world >= 1 && world <= 8 && rank >= 0 && rank < world, "bad arguments");
  ovg::PeerBarrierParams p{};
  for (int i = 0; i < world; ++i) {
    OVG_REQUIRE(flag_peers[i], "null flag array");
    p.flags[i] = flag_peers[i];
  }
  p.epoch = epoch_counter; p.rank = rank; p.world = world;
  ovg::peer_barrier_kernel<<<1, 32, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return post_launch("ovg_peer_barrier");
}

// layer: fp32 [K*T, 2C] export of the same half (ovg_aggregator_forward_layers), or NULL
static int inject_snapshot(float* x, const float* inj, void* slot, float* layer, float* cam_out, int K, int T, int C, int coff,
                           void* stream) {
  OVG_REQUIRE(x && K > 0 && T > 0 && C % 4 == 0, "bad arguments");
  OVG_REQUIRE(coff == 0 || coff == C, "coff must be 0 or C");
  ovg::InjectParams p{x, inj, reinterpret_cast<__nv_bfloat16*>(slot), cam_out, K, T, C, coff, layer};
  const int threads = C / 4 < 256 ? ((C / 4 + 31) / 32) * 32 : 256;
  ovg::inject_snapshot_kernel<<<(slot || layer) ? K * T : K, threads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return post_launch("ovg_inject_snapshot");
}

int ovg_inject_snapshot(float* x, const float* inj, void* slot, float* cam_out, int K, int T, int C, int coff,
                        void* stream) {
  return inject_snapshot(x, inj, slot, nullptr, cam_out, K, T, C, coff, stream);
}

int ovg_depth_im2col(const float* depth, const float* mask, const int* idx_stats, int n_stats, const int* idx_cols, int n_cols,
                     double* scratch, void* cols, int ldc, int B, int S, int H, int W, int patch, void* stream) {
  OVG_REQUIRE(depth && mask && idx_stats && scratch && (n_cols == 0 || (idx_cols && cols)), "null operand");
  OVG_REQUIRE(B > 0 && n_stats > 0 && n_stats <= S && n_cols >= 0 && n_cols <= S && H % patch == 0 && W % patch == 0 &&
                  patch % 2 == 0, "bad geometry");
  OVG_REQUIRE(ldc >= 2 * patch * patch && ldc % 2 == 0, "ldc too small / odd");
  OVG_REQUIRE((reinterpret_cast<uintptr_t>(depth) & 7) == 0 && (reinterpret_cast<uintptr_t>(mask) & 7) == 0 &&
                  (reinterpret_cast<uintptr_t>(cols) & 3) == 0, "depth / mask must be 8-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ovg::DepthParams ps{depth, mask, idx_stats, scratch, reinterpret_cast<__nv_bfloat16*>(cols), ldc, B, S, n_stats, H, W, patch};
  ovg::depth_stats_kernel<<<dim3(ovg::DEPTH_NCHUNK, B), 256, 0, st>>>(ps);
  int rc = post_launch("ovg_depth_im2col(stats)");
  if (rc) return rc;
  ovg::depth_scale_kernel<<<B, 256, 0, st>>>(ps);
  rc = post_launch("ovg_depth_im2col(scale)");
  if (rc || n_cols == 0) return rc;
  ovg::DepthParams pc = ps;
  pc.idx = idx_cols;
  pc.Sd = n_cols;
  if (patch == 14) ovg::depth_im2col_kernel<14><<<B * n_cols * (H / patch), 256, 0, st>>>(pc);
  else ovg::depth_im2col_kernel<0><<<B * n_cols * (H / patch), 256, 0, st>>>(pc);
  return post_launch("ovg_depth_im2col");
}

int ovg_image_im2col(const float* images, const float* mean3, const float* std3, void* cols, int ldc, int K, int H, int W,
                     int patch, void* stream) {
  OVG_REQUIRE(images && mean3 && std3 && cols, "null operand");
  OVG_REQUIRE(K > 0 && H % patch == 0 && W % patch == 0 && patch % 2 == 0 && ldc >= 3 * patch * patch && ldc % 8 == 0,
              "bad geometry");
  OVG_REQUIRE((reinterpret_cast<uintptr_t>(images) & 7) == 0, "images must be 8-byte aligned");
  ovg::ImageColParams p{images, reinterpret_cast<__nv_bfloat16*>(cols), ldc, K, H, W, patch, {}, {}};
  for (int c = 0; c < 3; ++c) {
    p.mean[c] = mean3[c];
    p.istd[c] = 1.0f / std3[c];
  }
  if (patch == 14) ovg::image_im2col_kernel<14><<<K * (H / patch), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  else ovg::image_im2col_kernel<0><<<K * (H / patch), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return post_launch("ovg_image_im2col");
}

int ovg_im2col3x3s2(const void* src, void* dst, int F, int h, int w, int C, void* stream) {
  OVG_REQUIRE(src && dst && F > 0 && h > 0 && w > 0 && C % 8 == 0, "bad arguments");
  const int oh = (h - 1) / 2 + 1, ow = (w - 1) / 2 + 1;
  ovg::Im2colParams p{reinterpret_cast<const __nv_bfloat16*>(src), reinterpret_cast<__nv_bfloat16*>(dst), F, h, w, C, oh, ow};
  const int threads = C / 8 < 128 ? ((C / 8 + 31) / 32) * 32 : 128;
  ovg::im2col3x3s2_kernel<<<dim3(F * oh * ow, 9), threads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return post_launch("ovg_im2col3x3s2");
}

int ovg_upsample_bilinear(const void* src, void* dst, const float* tx, const float* ty, int F, int h, int w, int H, int W,
                          int C, int f16, void* stream) {
  OVG_REQUIRE(src && dst && F > 0 && h > 0 && w > 0 && H > 0 && W > 0 && C % 16 == 0, "bad arguments");
  OVG_REQUIRE((tx == nullptr) == (ty == nullptr), "position tables come as a pair");
  OVG_REQUIRE(F <= 65535 && H + 2 <= 65535, "grid too large");
  ovg::UpsampleParams p{reinterpret_cast<const __nv_bfloat16*>(src), reinterpret_cast<__nv_bfloat16*>(dst), tx, ty,
                        F, h, w, H, W, C,
                        H > 1 ? static_cast<float>(h - 1) / static_cast<float>(H - 1) : 0.f,
                        W > 1 ? static_cast<float>(w - 1) / static_cast<float>(W - 1) : 0.f, f16 ? 1 : 0};
  const size_t row_smem = static_cast<size_t>(w) * 32 * sizeof(float);
  if (C % 32 == 0 && row_smem <= 48 * 1024 && C / 32 <= 65535) {
    dim3 grid(H + 2, F, C / 32);
    ovg::upsample_rows_kernel<<<grid, 256, row_smem, reinterpret_cast<cudaStream_t>(stream)>>>(p);
    return post_launch("ovg_upsample_bilinear");
  }
  const int per_row = (W + 2) * (C / 8);
  dim3 grid((per_row + 255) / 256, H + 2, F);
  ovg::upsample_bilinear_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return post_launch("ovg_upsample_bilinear");
}

int ovg_dpt_tail_supported(int h, int w, int H, int W, int C) {
  if (C != 128 || h < 2 || w < 2 || H < h || W < w) return 0;
  const float sx = W > 1 ? static_cast<float>(w - 1) / static_cast<float>(W - 1) : 0.f;
  const int span = static_cast<int>(sx * 129.0f) + 3;           // source pixels under 130 output pixels
  return span <= ovg::FT_VBUF_PX ? 1 : 0;
}

long long ovg_dpt_tail_scratch_bytes(int H, int W) { return (H > 0 && W > 0) ? 3LL * (H + W) * 32 * 4 : -1; }

int ovg_dpt_tail(const void* src, const float* tx, const float* ty, const void* w3x3, const float* bias, const float* w2,
                 const float* b2, int outc, int head_act, float* preds, float* conf, int F, int h, int w, int H, int W, int f16,
                 void* scratch, void* stream) {
  OVG_REQUIRE(src && w3x3 && bias && w2 && b2 && preds && conf, "null argument");
  OVG_REQUIRE((tx == nullptr) == (ty == nullptr), "position tables come as a pair");
  OVG_REQUIRE(tx == nullptr || (scratch && (reinterpret_cast<uintptr_t>(scratch) & 15) == 0),
              "position embedding needs 16-byte aligned scratch (ovg_dpt_tail_scratch_bytes)");
  OVG_REQUIRE(H >= 2 && W >= 2, "image too small");
  OVG_REQUIRE(F > 0 && outc >= 2 && outc <= 4, "bad arguments");
  OVG_REQUIRE(ovg_dpt_tail_supported(h, w, H, W, 128), "unsupported geometry (ovg_dpt_tail_supported)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  CUtensorMap tb;
  int rc = get_map(w3x3, 9 * 128, 32, 0, 9 * 128, 32, &tb);
  if (rc) return rc;
  ovg::TailParams p{};
  p.src = reinterpret_cast<const uint16_t*>(src);
  if (tx) {
    float* gx = static_cast<float*>(scratch);
    float* gy = gx + 3LL * W * 32;
    ovg::TailTableParams tp{tx, ty, reinterpret_cast<const uint16_t*>(w3x3), gx, gy, H, W, f16 ? 1 : 0};
    ovg::tail_tables_kernel<<<dim3(W > H ? W : H, 2), 96, 0, st>>>(tp);
    rc = post_launch("ovg_dpt_tail(tables)");
    if (rc) return rc;
    p.gx = gx; p.gy = gy;
  }
  p.bias = bias; p.w2 = w2; p.b2 = b2; p.preds = preds; p.conf = conf;
  p.F = F; p.h = h; p.w = w; p.H = H; p.W = W;
  p.sy = H > 1 ? static_cast<float>(h - 1) / static_cast<float>(H - 1) : 0.f;
  p.sx = W > 1 ? static_cast<float>(w - 1) / static_cast<float>(W - 1) : 0.f;
  p.outc = outc; p.head_act = head_act; p.f16 = f16 ? 1 : 0;
  p.n_strips = (W + 127) / 128;
  // segments of rows per (frame, strip): about three work items per SM, each paying two halo rows
  const int sms = num_sms();
  int segs = (3 * sms + F * p.n_strips - 1) / (F * p.n_strips);
  if (segs < 1) segs = 1;
  if (segs > H) segs = H;
  p.seg_rows = (H + segs - 1) / segs;
  if (p.seg_rows < 8 && H >= 8) p.seg_rows = 8;
  p.n_segs = (H + p.seg_rows - 1) / p.seg_rows;
  p.n_items = F * p.n_strips * p.n_segs;
  rc = p.f16 ? allow_dynamic_smem<ovg::fusedtail_kernel<true>>(ovg::FT_SMEM_BYTES)
             : allow_dynamic_smem<ovg::fusedtail_kernel<false>>(ovg::FT_SMEM_BYTES);
  if (rc) return rc;
  const int grid = p.n_items < sms ? p.n_items : sms;
  if (p.f16) ovg::fusedtail_kernel<true><<<grid, ovg::FT_THREADS, ovg::FT_SMEM_BYTES, st>>>(tb, p);
  else ovg::fusedtail_kernel<false><<<grid, ovg::FT_THREADS, ovg::FT_SMEM_BYTES, st>>>(tb, p);
  return post_launch("ovg_dpt_tail");
}

int ovg_preprocess_image_canvas(const unsigned char* src, int h, int w, int nw, int nh, int crop, int fh, const int* hmin,
                                const int* hcnt, const int* hk, int hksize, const int* vmin, const int* vcnt, const int* vk,
                                int vksize, unsigned char* tmp, float* out, int out_h, int out_w, int off_y, int off_x, float fill,
                                void* stream) {
  OVG_REQUIRE(src && out && h > 0 && w > 0 && nw > 0 && nh > 0 && crop >= 0 && fh > 0 && crop + fh <= nh, "bad geometry");
  OVG_REQUIRE(w == nw || (hmin && hcnt && hk && hksize > 0 && tmp), "horizontal pass needs its tap table and a temporary");
  OVG_REQUIRE(h == nh || (vmin && vcnt && vk && vksize > 0), "vertical pass needs its tap table");
  OVG_REQUIRE(off_y >= 0 && off_x >= 0 && off_y + fh <= out_h && off_x + nw <= out_w, "image does not fit its output frame");
  OVG_REQUIRE(h <= 65535 && out_h <= 65535, "image too tall");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const unsigned char* mid = src;
  if (w != nw) {
    ovg::ResizeParams ph{src, tmp, nullptr, hmin, hcnt, hk, hksize, h, w, nw, 0, 0, 0};
    ovg::resize_h_u8_kernel<<<dim3((nw + 127) / 128, h), 128, 0, st>>>(ph);
    int rc = post_launch("ovg_preprocess_image(horizontal)");
    if (rc) return rc;
    mid = tmp;
  }
  ovg::ResizeParams pv{mid, nullptr, out, vmin, vcnt, vk, vksize, h, w, nw, crop, fh, h == nh ? 1 : 0,
                       out_h, out_w, off_y, off_x, fill};
  ovg::resize_v_u8_f32_kernel<<<dim3((out_w + 127) / 128, out_h), 128, 0, st>>>(pv);
  return post_launch("ovg_preprocess_image");
}

int ovg_preprocess_image(const unsigned char* src, int h, int w, int nw, int nh, int crop, int fh, const int* hmin, const int* hcnt,
                         const int* hk, int hksize, const int* vmin, const int* vcnt, const int* vk, int vksize,
                         unsigned char* tmp, float* out, void* stream) {
  return ovg_preprocess_image_canvas(src, h, w, nw, nh, crop, fh, hmin, hcnt, hk, hksize, vmin, vcnt, vk, vksize, tmp, out, fh, nw,
                                     0, 0, 0.f, stream);
}

int ovg_preprocess_depth(const float* src, long long row_stride, long long col_stride, const int* sy, const int* sx, int crop,
                         int fh, int nw, float max_depth, float* depth, float* mask, void* stream) {
  OVG_REQUIRE(src && sy && sx && depth && mask && fh > 0 && nw > 0 && crop >= 0 && fh <= 65535, "bad arguments");
  ovg::DepthNearestParams p{src, row_stride, col_stride, sy, sx, depth, mask, crop, fh, nw, max_depth};
  ovg::depth_nearest_kernel<<<dim3((nw + 255) / 256, fh), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return post_launch("ovg_preprocess_depth");
}

int ovg_prepare_cameras(const float* c2w, const float* kin, const float* geom, const int* has, float* w2c, float* kout, int K,
                        void* stream) {
  OVG_REQUIRE(c2w && kin && geom && has && w2c && kout && K > 0, "bad arguments");
  ovg::CameraPrepParams p{c2w, kin, geom, has, w2c, kout, K};
  ovg::camera_prepare_kernel<<<(K + 63) / 64, 64, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return post_launch("ovg_prepare_cameras");
}

int ovg_pose_decode(const float* pose_enc, float* extrinsic, float* intrinsic, float* cam2world, int K, int H, int W,
                    void* stream) {
  OVG_REQUIRE(pose_enc && extrinsic && K > 0 && H > 0 && W > 0, "bad arguments");
  ovg::PoseDecodeParams p{pose_enc, extrinsic, intrinsic, cam2world, K, static_cast<float>(H), static_cast<float>(W)};
  ovg::pose_decode_kernel<<<(K + 127) / 128, 128, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return post_launch("ovg_pose_decode");
}

int ovg_unproject_depth(const float* depth, const float* intrinsic, const float* cam2world, float* world, int K, int H, int W,
                        void* stream) {
  OVG_REQUIRE(depth && intrinsic && cam2world && world && K > 0 && H > 0 && W > 0, "bad arguments");
  OVG_REQUIRE(K <= 65535, "too many frames");
  OVG_REQUIRE((reinterpret_cast<uintptr_t>(depth) & 15) == 0 && (reinterpret_cast<uintptr_t>(world) & 15) == 0,
              "depth / world must be 16-byte aligned");
  ovg::UnprojectParams p{depth, intrinsic, cam2world, world, K, H, W};
  const long long nq = (static_cast<long long>(H) * W + 3) / 4;
  int bx = static_cast<int>((nq + 255) / 256);
  const int cap = (num_sms() * 8 + K - 1) / K;       // ~8 blocks per SM over all frames, grid-stride inside
  if (bx > cap) bx = cap > 0 ? cap : 1;
  ovg::unproject_kernel<<<dim3(bx, K), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return post_launch("ovg_unproject_depth");
}

}  // extern "C"

namespace {

// Grid of the selection histograms and of the mask pass: one float4 per thread, at most 4 blocks per SM (grid-stride).
int select_blocks(long long n) {
  long long blocks = (n / 4 + 255) / 256;
  if (blocks > num_sms() * 4) blocks = num_sms() * 4;
  return blocks < 1 ? 1 : static_cast<int>(blocks);
}

// numpy.percentile(v[0, n), percent) (method "linear", exact) by radix select: one init launch, then 4 x (histogram, decide).
// workspace: OVG_PERCENTILE_WORKSPACE_BYTES (6 x u64 state | 512 x u32 histograms | ...); out3: device float[3] = the two
// neighbouring order statistics and the interpolated percentile.  count (optional) is zeroed by the init launch.
int radix_percentile(const float* v, long long n, float percent, void* workspace, float* out3, unsigned long long* count,
                     const std::string& what, cudaStream_t st) {
  // virtual index p/100 * (n - 1), linear interpolation between its two neighbours
  const double vi = static_cast<double>(percent) / 100.0 * static_cast<double>(n - 1);
  const unsigned long long r0 = static_cast<unsigned long long>(vi);
  const unsigned long long r1 = r0 + 1 < static_cast<unsigned long long>(n) ? r0 + 1 : r0;
  const double frac = vi - static_cast<double>(r0);
  unsigned long long* state = reinterpret_cast<unsigned long long*>(workspace);
  unsigned int* hist = reinterpret_cast<unsigned int*>(state + 6);
  ovg::select_init_kernel<<<1, 128, 0, st>>>(state, hist, r0, r1, count);
  int rc = post_launch((what + "(init)").c_str());
  if (rc) return rc;
  const int blocks = select_blocks(n);
  for (int pass = 0; pass < 4; ++pass) {
    ovg::SelectParams sp{v, n, state, hist, pass, out3, static_cast<float>(frac)};
    ovg::select_hist_kernel<<<blocks, 256, 0, st>>>(sp);
    rc = post_launch((what + "(hist)").c_str());
    if (rc) return rc;
    ovg::select_decide_kernel<<<1, 32, 0, st>>>(sp);
    rc = post_launch((what + "(decide)").c_str());
    if (rc) return rc;
  }
  return OVG_OK;
}

struct Arena {
  char* base;
  long long cap, off = 0;
  bool dry;        // size query: no pointers are formed
  Arena(void* b, long long c) : base(static_cast<char*>(b)), cap(c), dry(b == nullptr) {}
  void* take(long long bytes) {
    const long long at = (off + 255) & ~255LL;
    off = at + bytes;
    return dry ? nullptr : base + at;
  }
  template <typename T>
  T* get(long long n) { return static_cast<T*>(take(n * static_cast<long long>(sizeof(T)))); }
  bool ok() const { return dry || off <= cap; }
  long long bytes() const { return (off + 255) & ~255LL; }   // the layout's size in whole 256-byte blocks
};

// A caller's workspace for a layout of `need` bytes: non-null, `align`-byte aligned and at least `need` bytes long.
bool workspace_ok(const void* workspace, long long workspace_bytes, long long need, uintptr_t align) {
  return workspace && (reinterpret_cast<uintptr_t>(workspace) & (align - 1)) == 0 && workspace_bytes >= need;
}

// Point-cloud workspace, carved the same way by the size query and by every entry point.
struct CloudWorkspace {
  void* select;                      // OVG_PERCENTILE_WORKSPACE_BYTES
  float* sel;                        // [6][3] selection results of the scale
  double* center_partial;            // [CLOUD_CENTER_BLOCKS][3]
  unsigned int* tile_count;          // [tiles]
  unsigned long long* tile_offset;   // [tiles]
  long long bytes;
};

CloudWorkspace cloud_workspace(void* base, long long n) {
  Arena ar(base, 0);
  CloudWorkspace w;
  w.select = ar.take(OVG_PERCENTILE_WORKSPACE_BYTES);
  w.sel = ar.get<float>(18);
  w.center_partial = ar.get<double>(3LL * ovg::CLOUD_CENTER_BLOCKS);
  w.tile_count = ar.get<unsigned int>(ovg::compact_tiles(n));
  w.tile_offset = ar.get<unsigned long long>(ovg::compact_tiles(n));
  w.bytes = ar.bytes();
  return w;
}

}  // namespace

extern "C" {

int ovg_conf_percentile_mask(const float* conf, long long n, float percent, float floor_, void* workspace,
                             unsigned char* mask, float* threshold_out, unsigned long long* count_out, void* stream) {
  OVG_REQUIRE(conf && workspace && mask && threshold_out && n > 0, "bad arguments");
  OVG_REQUIRE(percent >= 0.f && percent <= 100.f, "percent must be in [0, 100]");
  OVG_REQUIRE((reinterpret_cast<uintptr_t>(conf) & 15) == 0 && (reinterpret_cast<uintptr_t>(mask) & 3) == 0 &&
                  (reinterpret_cast<uintptr_t>(workspace) & 15) == 0,
              "conf must be 16-byte, mask 4-byte, workspace 16-byte aligned");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // workspace: 6 x u64 state | 512 x u32 histograms | 3 x f32 results       (OVG_PERCENTILE_WORKSPACE_BYTES)
  float* res = reinterpret_cast<float*>(reinterpret_cast<unsigned int*>(reinterpret_cast<unsigned long long*>(workspace) + 6) + 512);
  int rc = radix_percentile(conf, n, percent, workspace, res, count_out, "ovg_conf_percentile_mask", st);
  if (rc) return rc;
  const int blocks = select_blocks(n);
  OVG_CUDA(cudaMemcpyAsync(threshold_out, res + 2, sizeof(float), cudaMemcpyDeviceToDevice, st));
  ovg::ConfMaskParams mp{conf, res + 2, mask, n, floor_, count_out};
  ovg::conf_mask_kernel<<<blocks, 256, 0, st>>>(mp);
  return post_launch("ovg_conf_percentile_mask");
}

long long ovg_point_cloud_workspace_bytes(long long n) { return n > 0 ? cloud_workspace(nullptr, n).bytes : -1; }

}  // extern "C"

namespace {

int cloud_params(const unsigned char* conf_mask, const float* images, int F, int H, int W, int mask_black_bg, int mask_white_bg,
                 void* workspace, long long workspace_bytes, ovg::CloudParams* p) {
  OVG_REQUIRE(conf_mask && images && workspace && F > 0 && H > 0 && W > 0, "bad arguments");
  const long long n = static_cast<long long>(F) * H * W;
  const CloudWorkspace w = cloud_workspace(workspace, n);
  OVG_REQUIRE(workspace_ok(workspace, workspace_bytes, w.bytes, 16),
              "workspace must be 16-byte aligned and ovg_point_cloud_workspace_bytes(F*H*W) long");
  OVG_REQUIRE(ovg::compact_tiles(n) < (1LL << 31), "too many pixels");
  *p = ovg::CloudParams{};
  p->conf_mask = conf_mask; p->images = images; p->n = n; p->hw = static_cast<long long>(H) * W;
  p->black_bg = mask_black_bg ? 1 : 0; p->white_bg = mask_white_bg ? 1 : 0;
  p->tile_count = w.tile_count; p->tile_offset = w.tile_offset;
  p->tiles = static_cast<int>(ovg::compact_tiles(n));
  return OVG_OK;
}

}  // namespace

extern "C" {

int ovg_point_cloud_count(const unsigned char* conf_mask, const float* images, int F, int H, int W, int mask_black_bg,
                          int mask_white_bg, void* workspace, long long workspace_bytes, unsigned long long* count_out,
                          void* stream) {
  OVG_REQUIRE(count_out, "null count_out");
  ovg::CloudParams p;
  int rc = cloud_params(conf_mask, images, F, H, W, mask_black_bg, mask_white_bg, workspace, workspace_bytes, &p);
  if (rc) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ovg::cloud_count_kernel<<<p.tiles, ovg::COMPACT_THREADS, 0, st>>>(p);
  rc = post_launch("ovg_point_cloud_count");
  if (rc) return rc;
  ovg::tile_scan_kernel<<<1, 1024, 0, st>>>(p.tile_count, p.tile_offset, count_out, p.tiles);
  return post_launch("ovg_point_cloud_count(scan)");
}

int ovg_point_cloud_gather(const float* points, const unsigned char* conf_mask, const float* images, int F, int H, int W,
                           int mask_black_bg, int mask_white_bg, int frame0, const void* workspace, long long workspace_bytes,
                           float* points_out, unsigned char* colors_out, int* frame_out, float* xyz, long long ld,
                           void* stream) {
  OVG_REQUIRE(points && points_out && colors_out && frame_out && xyz, "null operand");
  ovg::CloudParams p;
  int rc = cloud_params(conf_mask, images, F, H, W, mask_black_bg, mask_white_bg, const_cast<void*>(workspace),
                        workspace_bytes, &p);
  if (rc) return rc;
  OVG_REQUIRE(ld >= 0 && (ld % 4) == 0 && (reinterpret_cast<uintptr_t>(xyz) & 15) == 0,
              "xyz must be 16-byte aligned with a column stride ld % 4 == 0");
  p.points = points; p.frame0 = frame0;
  p.points_out = points_out; p.colors_out = colors_out; p.frame_out = frame_out; p.xyz = xyz; p.ld = ld;
  ovg::cloud_gather_kernel<<<p.tiles, ovg::COMPACT_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return post_launch("ovg_point_cloud_gather");
}

int ovg_point_cloud_center(const float* points, long long n, void* workspace, long long workspace_bytes, float* center_out,
                           void* stream) {
  OVG_REQUIRE(points && workspace && center_out && n > 0, "bad arguments");
  const CloudWorkspace w = cloud_workspace(workspace, n);
  OVG_REQUIRE(workspace_ok(workspace, workspace_bytes, w.bytes, 16),
              "workspace must be 16-byte aligned and ovg_point_cloud_workspace_bytes(n) long");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ovg::CloudCenterParams p{points, n, w.center_partial, center_out};
  ovg::cloud_center_partial_kernel<<<ovg::CLOUD_CENTER_BLOCKS, 256, 0, st>>>(p);
  int rc = post_launch("ovg_point_cloud_center");
  if (rc) return rc;
  ovg::cloud_center_final_kernel<<<1, 32, 0, st>>>(p);
  return post_launch("ovg_point_cloud_center(final)");
}

int ovg_point_cloud_scale(const float* xyz, long long n_kept, long long ld, void* workspace, long long workspace_bytes,
                          float* scale_out, void* stream) {
  OVG_REQUIRE(xyz && workspace && scale_out && n_kept > 0 && ld >= n_kept && ld % 4 == 0, "bad arguments");
  OVG_REQUIRE((reinterpret_cast<uintptr_t>(xyz) & 15) == 0, "xyz must be 16-byte aligned");
  const CloudWorkspace w = cloud_workspace(workspace, 1);   // the scale uses only the fixed-size head of the workspace
  OVG_REQUIRE(workspace_ok(workspace, workspace_bytes, w.bytes, 16),
              "workspace must be 16-byte aligned and ovg_point_cloud_workspace_bytes() long");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  for (int q = 0; q < 2; ++q)
    for (int a = 0; a < 3; ++a) {
      const int rc = radix_percentile(xyz + a * ld, n_kept, q ? 95.f : 5.f, w.select, w.sel + (q * 3 + a) * 3, nullptr,
                                      "ovg_point_cloud_scale", st);
      if (rc) return rc;
    }
  ovg::cloud_scale_kernel<<<1, 32, 0, st>>>(w.sel, scale_out);
  return post_launch("ovg_point_cloud_scale");
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------- reciprocal matches
namespace {

// Match workspace, carved the same way by the size query and by every entry point.
struct MatchWorkspace {
  ovg::MatchParams p;
  int passes;          // 8-bit radix-sort passes over the cell ids
  long long bytes;
};

MatchWorkspace match_workspace(void* base, int V, long long cap, int P) {
  Arena ar(base, 0);
  MatchWorkspace w;
  ovg::MatchParams& p = w.p;
  p = ovg::MatchParams{};
  p.V = V; p.cap = cap; p.P = P;
  p.tiles = static_cast<int>(ovg::compact_tiles(cap));
  p.ptiles = p.tiles;
  p.cells_cap = ovg::match_cells_cap(cap);
  p.flag = ar.get<unsigned int>(1);
  p.hist = ar.get<unsigned int>(3LL * V * ovg::MATCH_BINS);
  p.grid = ar.get<ovg::MatchGrid>(V);
  p.range0 = ar.get<float>(6LL * V);
  p.view_tile_count = ar.get<unsigned int>(static_cast<long long>(V) * p.tiles);
  p.view_tile_offset = ar.get<unsigned int>(static_cast<long long>(V) * p.tiles);
  p.pts = ar.get<float4>(V * cap);
  p.rtiles = static_cast<int>((cap + ovg::MATCH_RADIX_TILE - 1) / ovg::MATCH_RADIX_TILE);
  for (int b = 0; b < 2; ++b) {
    p.keys[b] = ar.get<int>(V * cap);
    p.vals[b] = ar.get<float4>(V * cap);
  }
  p.radix_off = ar.get<unsigned int>(256LL * V * p.rtiles);
  int bits = 0;
  while ((1LL << bits) < p.cells_cap) ++bits;
  w.passes = (bits + 7) / 8;
  p.sorted = p.vals[w.passes & 1];
  p.cell_count = ar.get<int>(V * p.cells_cap);
  p.cell_start = ar.get<int>(V * (p.cells_cap + 1));
  p.nn = ar.get<int>(2LL * P * cap);
  p.pair_tile_count = ar.get<unsigned int>(static_cast<long long>(P) * p.ptiles);
  p.pair_tile_offset = ar.get<unsigned long long>(static_cast<long long>(P) * p.ptiles);
  p.total = ar.get<unsigned long long>(1);
  w.bytes = ar.bytes();
  return w;
}

int match_check(int V, long long cap, int P, const void* workspace, long long workspace_bytes, ovg::MatchParams* p,
                int* passes = nullptr) {
  // cap < 2^30 keeps the cell ids (cells_cap = 2 cap + 64) and the slots inside a view in int range
  OVG_REQUIRE(V > 0 && V <= 65535 && cap > 0 && cap < (1LL << 30) && P > 0 && 2LL * P <= 65535, "bad sizes");
  OVG_REQUIRE(static_cast<long long>(V) * cap < (1LL << 40), "too many points");
  const MatchWorkspace w = match_workspace(const_cast<void*>(workspace), V, cap, P);
  OVG_REQUIRE(workspace_ok(workspace, workspace_bytes, w.bytes, 256),
              "workspace must be 256-byte aligned and ovg_match_workspace_bytes(V, cap, P) long");
  *p = w.p;
  if (passes) *passes = w.passes;
  return OVG_OK;
}

// grid-stride blocks over one view's points, per view
int match_blocks(long long cap) {
  const long long b = (cap + 255) / 256;
  return static_cast<int>(b < 64 ? (b < 1 ? 1 : b) : 64);
}

}  // namespace

extern "C" {

long long ovg_match_workspace_bytes(int V, long long cap, int P) {
  return (V > 0 && cap > 0 && P > 0) ? match_workspace(nullptr, V, cap, P).bytes : -1;
}

int ovg_match_index(const float* points, const unsigned char* keep, int V, long long cap, int P, void* workspace,
                    long long workspace_bytes, void* stream) {
  ovg::MatchParams p;
  int passes = 0;
  int rc = match_check(V, cap, P, workspace, workspace_bytes, &p, &passes);
  if (rc) return rc;
  OVG_REQUIRE(points, "null points");
  p.points = points;
  p.keep = keep;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  OVG_CUDA(cudaMemsetAsync(p.flag, 0, 4, st));
  OVG_CUDA(cudaMemsetAsync(p.hist, 0, 4LL * V * 3 * ovg::MATCH_BINS, st));
  OVG_CUDA(cudaMemsetAsync(p.cell_count, 0, 4LL * V * p.cells_cap, st));
  ovg::match_keep_count_kernel<<<dim3(p.tiles, V), ovg::COMPACT_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_match_index(keep count)"))) return rc;
  ovg::match_keep_scan_kernel<<<V, 1024, 0, st>>>(p);
  if ((rc = post_launch("ovg_match_index(keep scan)"))) return rc;
  ovg::match_keep_gather_kernel<<<dim3(p.tiles, V), ovg::COMPACT_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_match_index(keep gather)"))) return rc;
  const dim3 grid(match_blocks(cap), V);
  for (int pass = 0; pass < 2; ++pass) {
    ovg::match_hist_kernel<<<grid, 256, 0, st>>>(p, pass);
    if ((rc = post_launch("ovg_match_index(histogram)"))) return rc;
    ovg::match_range_kernel<<<V, 32, 0, st>>>(p, pass);
    if ((rc = post_launch("ovg_match_index(range)"))) return rc;
  }
  ovg::match_cell_count_kernel<<<grid, 256, 0, st>>>(p);
  if ((rc = post_launch("ovg_match_index(cell count)"))) return rc;
  ovg::match_cell_scan_kernel<<<V, 1024, 0, st>>>(p);
  if ((rc = post_launch("ovg_match_index(cell scan)"))) return rc;
  const dim3 rgrid(p.rtiles, V);
  for (int pass = 0; pass < passes; ++pass) {
    ovg::match_radix_count_kernel<<<rgrid, ovg::MATCH_RADIX_TILE, 0, st>>>(p, 8 * pass, pass & 1);
    if ((rc = post_launch("ovg_match_index(radix count)"))) return rc;
    ovg::match_radix_scan_kernel<<<V, 1024, 0, st>>>(p);
    if ((rc = post_launch("ovg_match_index(radix scan)"))) return rc;
    ovg::match_radix_scatter_kernel<<<rgrid, ovg::MATCH_RADIX_TILE, 0, st>>>(p, 8 * pass, pass & 1);
    if ((rc = post_launch("ovg_match_index(radix scatter)"))) return rc;
  }
  return OVG_OK;
}

int ovg_match_query(const int* pairs, int P, int V, long long cap, void* workspace, long long workspace_bytes, long long* counts_out,
                    void* stream) {
  ovg::MatchParams p;
  int rc = match_check(V, cap, P, workspace, workspace_bytes, &p);
  if (rc) return rc;
  OVG_REQUIRE(pairs && counts_out, "null pairs / counts_out");
  OVG_REQUIRE(static_cast<long long>(P) * p.ptiles < (1LL << 31), "too many pairs");
  p.pairs = pairs;
  p.counts = counts_out;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ovg::match_query_kernel<<<dim3(static_cast<unsigned>((cap + ovg::MATCH_QUERY_THREADS - 1) / ovg::MATCH_QUERY_THREADS), 2 * P),
                            ovg::MATCH_QUERY_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_match_query"))) return rc;
  ovg::match_recip_count_kernel<<<dim3(p.ptiles, P), ovg::COMPACT_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_match_query(reciprocal count)"))) return rc;
  ovg::tile_scan_kernel<<<1, 1024, 0, st>>>(p.pair_tile_count, p.pair_tile_offset, p.total,
                                            static_cast<long long>(P) * p.ptiles);
  if ((rc = post_launch("ovg_match_query(scan)"))) return rc;
  ovg::match_counts_kernel<<<(P + 1 + 255) / 256, 256, 0, st>>>(p);
  return post_launch("ovg_match_query(counts)");
}

int ovg_match_gather(const int* pairs, int P, int V, long long cap, int W, const void* workspace, long long workspace_bytes,
                     long long* xy_i, long long* xy_j, void* stream) {
  ovg::MatchParams p;
  int rc = match_check(V, cap, P, workspace, workspace_bytes, &p);
  if (rc) return rc;
  OVG_REQUIRE(pairs && xy_i && xy_j && W > 0, "bad arguments");
  p.pairs = pairs;
  ovg::MatchOut o{W, xy_i, xy_j, -1, nullptr, nullptr};
  ovg::match_gather_kernel<<<dim3(p.ptiles, P), ovg::COMPACT_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p, o);
  return post_launch("ovg_match_gather");
}

int ovg_match_pair(const int* pairs, int P, int V, long long cap, int pair, const void* workspace, long long workspace_bytes,
                   unsigned char* reciprocal, long long* nn, void* stream) {
  ovg::MatchParams p;
  int rc = match_check(V, cap, P, workspace, workspace_bytes, &p);
  if (rc) return rc;
  OVG_REQUIRE(pairs && reciprocal && nn && pair >= 0 && pair < P, "bad arguments");
  p.pairs = pairs;
  ovg::MatchOut o{1, nullptr, nullptr, pair, reciprocal, nn};
  ovg::match_pair_kernel<<<static_cast<unsigned>((cap + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p, o);
  return post_launch("ovg_match_pair");
}

}  // extern "C"

// -------------------------------------------------------------------------------------------------------------- triangle mesh
namespace {

// Mesh workspace, carved the same way by the size query and by every entry point.
ovg::MeshParams mesh_workspace(void* base, int F, int H, int W, long long* bytes) {
  Arena ar(base, 0);
  ovg::MeshParams p{};
  p.H = H; p.W = W;
  p.hw = static_cast<long long>(H) * W;
  p.n = F * p.hw;
  p.tpv = static_cast<int>(ovg::compact_tiles(p.hw));
  p.T = F * p.tpv;
  p.keep = ar.get<unsigned char>(p.n);
  p.remap = ar.get<int>(p.n);
  p.tile_count = ar.get<unsigned int>(static_cast<long long>(ovg::MESH_STREAMS) * p.T);
  p.tile_offset = ar.get<unsigned long long>(static_cast<long long>(ovg::MESH_STREAMS) * p.T + 1);
  *bytes = ar.bytes();
  return p;
}

int mesh_check(int F, int H, int W, const void* workspace, long long workspace_bytes, ovg::MeshParams* p) {
  OVG_REQUIRE(F > 0 && F <= 65535 && H > 0 && W > 0, "bad sizes");
  OVG_REQUIRE(static_cast<long long>(F) * H * W < (1LL << 31), "F*H*W must be below 2^31");
  long long bytes = 0;
  *p = mesh_workspace(const_cast<void*>(workspace), F, H, W, &bytes);
  OVG_REQUIRE(workspace_ok(workspace, workspace_bytes, bytes, 256),
              "workspace must be 256-byte aligned and ovg_mesh_workspace_bytes(F, H, W) long");
  return OVG_OK;
}

}  // namespace

extern "C" {

long long ovg_mesh_workspace_bytes(int F, int H, int W) {
  if (F <= 0 || H <= 0 || W <= 0) return -1;
  long long bytes = 0;
  mesh_workspace(nullptr, F, H, W, &bytes);
  return bytes;
}

int ovg_mesh_count(const unsigned char* conf_mask, const float* images, int F, int H, int W, int mask_black_bg,
                   int mask_white_bg, void* workspace, long long workspace_bytes, long long* counts_out, void* stream) {
  ovg::MeshParams p;
  int rc = mesh_check(F, H, W, workspace, workspace_bytes, &p);
  if (rc) return rc;
  OVG_REQUIRE(conf_mask && counts_out, "null conf_mask / counts_out");
  OVG_REQUIRE(images || !(mask_black_bg || mask_white_bg), "the background masks need images");
  p.conf_mask = conf_mask; p.images = images;
  p.black_bg = mask_black_bg ? 1 : 0; p.white_bg = mask_white_bg ? 1 : 0;
  p.totals = counts_out;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ovg::mesh_keep_kernel<<<static_cast<unsigned>((p.n + 255) / 256), 256, 0, st>>>(p);
  if ((rc = post_launch("ovg_mesh_count(keep)"))) return rc;
  ovg::mesh_count_kernel<<<dim3(p.tpv, F), ovg::COMPACT_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_mesh_count"))) return rc;
  const long long tiles = static_cast<long long>(ovg::MESH_STREAMS) * p.T;
  ovg::tile_scan_kernel<<<1, 1024, 0, st>>>(p.tile_count, p.tile_offset, p.tile_offset + tiles, tiles);
  if ((rc = post_launch("ovg_mesh_count(scan)"))) return rc;
  ovg::mesh_totals_kernel<<<1, 32, 0, st>>>(p);
  return post_launch("ovg_mesh_count(totals)");
}

int ovg_mesh_faces(const float* images, const void* colors, int color_bytes, int F, int H, int W, const void* workspace,
                   long long workspace_bytes, long long* faces, void* face_colors, void* stream) {
  ovg::MeshParams p;
  int rc = mesh_check(F, H, W, workspace, workspace_bytes, &p);
  if (rc) return rc;
  OVG_REQUIRE(faces && face_colors, "null faces / face_colors");
  OVG_REQUIRE(images || (colors && (color_bytes == 1 || color_bytes == 2 || color_bytes == 4 || color_bytes == 8)),
              "face colours need images, or colors with color_bytes 1, 2, 4 or 8");
  p.images = images; p.colors = colors; p.color_bytes = color_bytes;
  p.faces = faces; p.face_colors = face_colors;
  ovg::mesh_faces_kernel<<<dim3(p.tpv, F), ovg::COMPACT_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return post_launch("ovg_mesh_faces");
}

int ovg_mesh_compact(const float* points, const float* images, int F, int H, int W, const void* workspace,
                     long long workspace_bytes, float* positions, unsigned char* colors, int* indices, void* stream) {
  ovg::MeshParams p;
  int rc = mesh_check(F, H, W, workspace, workspace_bytes, &p);
  if (rc) return rc;
  OVG_REQUIRE(points && images && positions && colors && indices, "null operand");
  p.points = points; p.images = images;
  p.positions = positions; p.vertex_colors = colors; p.indices = indices;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ovg::mesh_vertices_kernel<<<dim3(p.tpv, F), ovg::COMPACT_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_mesh_compact(vertices)"))) return rc;
  ovg::mesh_indices_kernel<<<dim3(p.tpv, F), ovg::COMPACT_THREADS, 0, st>>>(p);
  return post_launch("ovg_mesh_compact(indices)");
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------- sky segmentation
namespace {

// Sky workspace, carved the same way by the size query and by the entry point.
ovg::SkyParams sky_workspace(void* base, int F, int H, int W, long long* bytes) {
  Arena ar(base, 0);
  ovg::SkyParams p{};
  p.F = F; p.H = H; p.W = W;
  p.hw = static_cast<long long>(H) * W;
  p.n = F * p.hw;
  p.tiles_x = (W + ovg::SKY_TILE - 1) / ovg::SKY_TILE;
  p.label = ar.get<int>(p.n);
  p.area = ar.get<int>(p.n);
  p.view_max = ar.get<int>(F);
  *bytes = ar.bytes();
  return p;
}

}  // namespace

extern "C" {

long long ovg_sky_workspace_bytes(int F, int H, int W) {
  if (F <= 0 || H <= 0 || W <= 0) return -1;
  long long bytes = 0;
  sky_workspace(nullptr, F, H, W, &bytes);
  return bytes;
}

int ovg_segment_sky(const void* image, int image_u8, long long view_stride, long long pixel_stride, long long channel_stride,
                    int F, int H, int W, const float* conf, void* workspace, long long workspace_bytes, unsigned char* sky_out,
                    float* conf_out, void* stream) {
  OVG_REQUIRE(F > 0 && F <= 65535 && H > 0 && W > 0, "bad sizes");
  OVG_REQUIRE(static_cast<long long>(F) * H * W < (1LL << 31), "F*H*W must be below 2^31");
  OVG_REQUIRE(image && sky_out && (conf == nullptr) == (conf_out == nullptr), "null image / sky_out, or conf without conf_out");
  long long bytes = 0;
  ovg::SkyParams p = sky_workspace(workspace, F, H, W, &bytes);
  OVG_REQUIRE(workspace_ok(workspace, workspace_bytes, bytes, 256),
              "workspace must be 256-byte aligned and ovg_sky_workspace_bytes(F, H, W) long");
  p.image = image; p.u8 = image_u8 ? 1 : 0;
  p.view_stride = view_stride; p.pixel_stride = pixel_stride; p.channel_stride = channel_stride;
  p.conf = conf; p.conf_out = conf_out; p.sky = sky_out;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int tiles = p.tiles_x * ((H + ovg::SKY_TILE - 1) / ovg::SKY_TILE);
  ovg::sky_open_kernel<<<dim3(tiles, F), ovg::SKY_THREADS, 0, st>>>(p);
  int rc = post_launch("ovg_segment_sky(colour test, opening)");
  if (rc) return rc;
  const unsigned blocks = static_cast<unsigned>((p.n + 255) / 256);
  ovg::sky_merge_kernel<<<blocks, 256, 0, st>>>(p);
  if ((rc = post_launch("ovg_segment_sky(merge)"))) return rc;
  ovg::sky_area_kernel<<<blocks, 256, 0, st>>>(p);
  if ((rc = post_launch("ovg_segment_sky(area)"))) return rc;
  ovg::sky_max_kernel<<<blocks, 256, 0, st>>>(p);
  if ((rc = post_launch("ovg_segment_sky(max area)"))) return rc;
  ovg::sky_select_kernel<<<blocks, 256, 0, st>>>(p);
  return post_launch("ovg_segment_sky(select)");
}

int ovg_sky_mask_conf(const float* conf, const unsigned char* sky, long long n, float* conf_out, void* stream) {
  OVG_REQUIRE(conf && sky && conf_out && n > 0 && n < (1LL << 40), "bad arguments");
  ovg::sky_mask_conf_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      conf, sky, n, conf_out);
  return post_launch("ovg_sky_mask_conf");
}

}  // extern "C"

// -------------------------------------------------------------------------------------------------- farthest point sampling
namespace {

// FPS workspace, carved the same way by the size query and by the entry point.
ovg::FpsParams fps_workspace(void* base, int B, long long N, long long* bytes) {
  Arena ar(base, 0);
  ovg::FpsParams p{};
  p.B = B; p.N = N;
  p.arrive = ar.get<unsigned>(B);
  p.slots = ar.get<ovg::FpsSlot>(2LL * ovg::FPS_MAX_CTAS);
  p.dist = ar.get<float>(static_cast<long long>(B) * N);
  *bytes = ar.bytes();
  return p;
}

}  // namespace

extern "C" {

long long ovg_fps_workspace_bytes(int B, long long N) {
  if (B <= 0 || N <= 0) return -1;
  long long bytes = 0;
  fps_workspace(nullptr, B, N, &bytes);
  return bytes;
}

int ovg_farthest_point_sample(const float* xyz, int B, long long N, int npoint, const long long* start, int include_ends,
                              void* workspace, long long workspace_bytes, long long* inds_out, void* stream) {
  OVG_REQUIRE(B > 0 && N > 0 && npoint > 0, "bad sizes");
  OVG_REQUIRE(N < (1LL << 31), "N must be below 2^31");
  OVG_REQUIRE(npoint <= N, "npoint must be <= N");
  OVG_REQUIRE(static_cast<long long>(B) * N < (1LL << 40), "too many points");
  OVG_REQUIRE(xyz && inds_out && (start || include_ends), "null xyz / inds_out, or no start without include_ends");
  long long bytes = 0;
  ovg::FpsParams p = fps_workspace(workspace, B, N, &bytes);
  OVG_REQUIRE(workspace_ok(workspace, workspace_bytes, bytes, 256),
              "workspace must be 256-byte aligned and ovg_fps_workspace_bytes(B, N) long");
  p.xyz = xyz; p.start = start; p.inds = inds_out; p.npoint = npoint; p.ends = include_ends ? 1 : 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (N <= ovg::FPS_CTA_POINTS) {   // one CTA per batch, every point in its shared memory
    int rc = allow_dynamic_smem<ovg::fps_cta_kernel>(ovg::FPS_SMEM_BYTES);
    if (rc) return rc;
    ovg::fps_cta_kernel<<<B, ovg::FPS_THREADS, static_cast<int>(N) * 16, st>>>(p);
    return post_launch("ovg_farthest_point_sample(cta)");
  }
  // The grid kernel spins on the other CTAs of its group: launched cooperatively, sized by the occupancy query, so the
  // launch fails rather than run with CTAs that are not co-resident.
  int rc = allow_dynamic_smem<ovg::fps_grid_kernel>(ovg::FPS_SMEM_BYTES);
  if (rc) return rc;
  int per_sm = 0;
  OVG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ovg::fps_grid_kernel, ovg::FPS_THREADS,
                                                         ovg::FPS_SMEM_BYTES));
  OVG_REQUIRE(per_sm > 0, "the grid kernel does not fit on an SM");
  const int grid = std::min(per_sm * num_sms(), ovg::FPS_MAX_CTAS);
  p.groups = std::min(B, grid);
  p.G = grid / p.groups;
  OVG_CUDA(cudaMemsetAsync(p.arrive, 0, sizeof(unsigned) * B, st));
  void* args[] = {&p};
  OVG_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(ovg::fps_grid_kernel), dim3(grid), dim3(ovg::FPS_THREADS), args,
                                       ovg::FPS_SMEM_BYTES, st));
  return post_launch("ovg_farthest_point_sample(grid)");
}

}  // extern "C"

// ----------------------------------------------------------------------------------------------------------- image ranking
namespace {

// Ranking workspace, carved the same way by the size query and by the entry point: the packed operands, and on the grid
// path one scratch of two key / index buffers per CTA.
ovg::RankParams ranking_workspace(void* base, long long N, int out_f64, long long* bytes) {
  Arena ar(base, 0);
  ovg::RankParams p{};
  p.pose = ar.get<double>(N * 12);
  if (N > ovg::RANK_CTA_VIEWS) {
    p.scratch_stride = (N * (2 * (out_f64 ? 8 : 4) + 8) + 255) & ~255LL;
    p.scratch = ar.get<unsigned char>(ovg::RANK_GRID_CTAS * p.scratch_stride);
  }
  *bytes = ar.bytes();
  return p;
}

template <typename T, typename K>
int launch_ranking(const ovg::RankParams& p, cudaStream_t st) {
  if (p.N <= ovg::RANK_CTA_VIEWS) {
    const int smem = p.N * static_cast<int>(2 * sizeof(K) + 8);
    const int rc = allow_dynamic_smem<ovg::rank_smem_kernel<T, K>>(ovg::RANK_CTA_VIEWS * static_cast<int>(2 * sizeof(K) + 8));
    if (rc) return rc;
    ovg::rank_smem_kernel<T, K><<<p.N, ovg::RANK_THREADS, smem, st>>>(p);
    return post_launch("ovg_compute_ranking(smem)");
  }
  ovg::rank_grid_kernel<T, K><<<ovg::RANK_GRID_CTAS, ovg::RANK_THREADS, 0, st>>>(p);
  return post_launch("ovg_compute_ranking(grid)");
}

}  // namespace

extern "C" {

long long ovg_ranking_workspace_bytes(long long N, int out_f64) {
  if (N <= 0 || N >= (1LL << 31)) return -1;
  long long bytes = 0;
  ranking_workspace(nullptr, N, out_f64, &bytes);
  return bytes;
}

int ovg_compute_ranking(const void* extrinsics, int in_f64, long long N, long long view_stride, long long row_stride,
                        long long col_stride, double lambda_t, int normalize, int out_f64, long long k, void* workspace,
                        long long workspace_bytes, long long* ranking, void* dists, void* stream) {
  OVG_REQUIRE(N > 0 && N < (1LL << 31), "N must be in [1, 2^31)");
  OVG_REQUIRE(k >= 1 && k <= N, "k must be in [1, N]");
  OVG_REQUIRE(extrinsics && ranking && dists, "null extrinsics / ranking / dists");
  long long bytes = 0;
  ovg::RankParams p = ranking_workspace(workspace, N, out_f64, &bytes);
  OVG_REQUIRE(workspace_ok(workspace, workspace_bytes, bytes, 256),
              "workspace must be 256-byte aligned and ovg_ranking_workspace_bytes(N, out_f64) long");
  p.ext = extrinsics; p.s0 = view_stride; p.s1 = row_stride; p.s2 = col_stride;
  p.ranking = ranking; p.dists = dists; p.lambda = lambda_t;
  p.N = static_cast<int>(N); p.k = static_cast<int>(k);
  p.in_f64 = in_f64 ? 1 : 0; p.out_f64 = out_f64 ? 1 : 0; p.normalize = normalize ? 1 : 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ovg::rank_prep_kernel<<<1, ovg::RANK_PREP_THREADS, 0, st>>>(p);
  const int rc = post_launch("ovg_compute_ranking(prep)");
  if (rc) return rc;
  return p.out_f64 ? launch_ranking<double, unsigned long long>(p, st) : launch_ranking<float, unsigned>(p, st);
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------- JPEG decode
struct ovg_jpeg_plan : ovg::jpg::Plan {};

extern "C" {

int ovg_jpeg_plan_create(const unsigned char* const* files, const long long* nbytes, int n, int subseq_bits,
                         ovg_jpeg_plan** plan) {
  OVG_REQUIRE(plan && n >= 0 && (n == 0 || (files && nbytes)), "bad arguments");
  OVG_REQUIRE(subseq_bits == 0 || (subseq_bits >= ovg::jpg::MIN_SUBSEQ_BITS && subseq_bits <= ovg::jpg::MAX_SUBSEQ_BITS),
              "subseq_bits must be 0 or in [OVG_JPEG_MIN_SUBSEQ_BITS, 65536]");
  ovg_jpeg_plan* out = nullptr;
  try {
    out = new ovg_jpeg_plan;
    ovg::jpg::plan_build(out, files, nbytes, n, subseq_bits);
  } catch (const std::exception& e) {
    delete out;
    return fail(OVG_E_INVALID, std::string("ovg_jpeg_plan_create: ") + e.what());
  }
  *plan = out;
  return OVG_OK;
}

void ovg_jpeg_plan_destroy(ovg_jpeg_plan* plan) { delete plan; }

int ovg_jpeg_plan_file(const ovg_jpeg_plan* plan, int i, int* route, int* width, int* height, int* ncomp) {
  OVG_REQUIRE(plan && i >= 0 && i < static_cast<int>(plan->route.size()), "bad file index");
  if (route) *route = plan->route[i];
  if (width) *width = plan->width[i];
  if (height) *height = plan->height[i];
  if (ncomp) *ncomp = plan->ncomp[i];
  return OVG_OK;
}

long long ovg_jpeg_plan_stream_bytes(const ovg_jpeg_plan* plan) { return plan ? plan->stream_bytes : -1; }
long long ovg_jpeg_plan_subsequences(const ovg_jpeg_plan* plan) { return plan ? plan->nsub : -1; }
long long ovg_jpeg_plan_segments(const ovg_jpeg_plan* plan) { return plan ? static_cast<long long>(plan->segs.size()) : -1; }
int ovg_jpeg_plan_rounds(const ovg_jpeg_plan* plan) { return plan ? plan->rounds : -1; }

long long ovg_jpeg_plan_workspace_bytes(const ovg_jpeg_plan* plan) {
  return plan ? ovg::jpg::plan_workspace(plan, static_cast<int>(plan->route.size()), nullptr).bytes : -1;
}

int ovg_jpeg_plan_segment(const ovg_jpeg_plan* plan, long long k, int* file, long long* offset, long long* nbytes, int* first_mcu,
                          int* n_mcu) {
  OVG_REQUIRE(plan && k >= 0 && k < static_cast<long long>(plan->segs.size()), "bad segment index");
  const ovg::jpg::HostSeg& s = plan->segs[k];
  if (file) *file = plan->files[s.file].out_index;
  if (offset) *offset = plan->data_off + s.byte_off;
  if (nbytes) *nbytes = s.nbytes;
  if (first_mcu) *first_mcu = s.first_mcu;
  if (n_mcu) *n_mcu = s.n_mcu;
  return OVG_OK;
}

int ovg_jpeg_plan_fill_stream(const ovg_jpeg_plan* plan, void* dst) {
  OVG_REQUIRE(plan && (dst || plan->stream_bytes == 0), "bad arguments");
  ovg::jpg::plan_fill(plan, static_cast<uint8_t*>(dst));
  return OVG_OK;
}

int ovg_jpeg_decode(ovg_jpeg_plan* plan, const void* d_stream, unsigned char* const* d_out, unsigned* d_status, void* workspace,
                    long long workspace_bytes, void* stream) {
  using namespace ovg::jpg;
  OVG_REQUIRE(plan && d_status, "bad arguments");
  const int n = static_cast<int>(plan->route.size());
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (n) OVG_CUDA(cudaMemsetAsync(d_status, 0, sizeof(unsigned) * n, st));
  plan->rounds = 0;
  if (plan->files.empty()) return OVG_OK;
  OVG_REQUIRE(d_stream && d_out && workspace && (reinterpret_cast<uintptr_t>(d_stream) & 255) == 0 &&
              (reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "stream and workspace must be 256-byte aligned");
  const Workspace w = plan_workspace(plan, n, workspace);
  OVG_REQUIRE(workspace_bytes >= w.bytes, "workspace smaller than ovg_jpeg_plan_workspace_bytes()");
  for (const FileDev& f : plan->files) OVG_REQUIRE(d_out[f.out_index], "null output for a device-routed file");
  const uint8_t* base = static_cast<const uint8_t*>(d_stream);
  Params p;
  p.files = reinterpret_cast<const FileDev*>(base + plan->files_off);
  p.segs = reinterpret_cast<const SegDev*>(base + plan->segs_off);
  p.huffs = reinterpret_cast<const Huff*>(base + plan->huffs_off);
  p.data = base + plan->data_off;
  p.nfiles = static_cast<int>(plan->files.size());
  p.nsegs = static_cast<int>(plan->segs.size());
  p.nsub = plan->nsub; p.nblocks = plan->nblocks; p.npix = plan->npix;
  p.subseq_bits = plan->subseq_bits;
  p.exits = w.exits; p.counts = w.counts; p.pre = w.pre; p.chunk = w.chunk; p.coef = w.coef;
  p.dc_agg = w.dc_agg; p.dc_aggf = w.dc_aggf; p.dc_head = w.dc_head; p.planes = w.planes; p.out = w.out;
  p.status = d_status; p.changed = w.changed;
  OVG_CUDA(cudaMemcpyAsync(w.out, d_out, sizeof(void*) * n, cudaMemcpyHostToDevice, st));
  OVG_CUDA(cudaMemsetAsync(w.exits, 0, 4 * plan->nsub, st));
  // sync rounds: each round fixes at least one more subsequence, so at most nsub + 1 rounds
  const unsigned sub_grid = static_cast<unsigned>((plan->nsub + 255) / 256);
  for (long long r = 0; r <= plan->nsub; ++r) {
    OVG_CUDA(cudaMemsetAsync(w.changed, 0, 4, st));
    jpeg_sync_kernel<<<sub_grid, 256, 0, st>>>(p);
    int rc = post_launch("ovg_jpeg_decode(sync)");
    if (rc) return rc;
    int changed = 0;
    OVG_CUDA(cudaMemcpyAsync(&changed, w.changed, 4, cudaMemcpyDeviceToHost, st));
    OVG_CUDA(cudaStreamSynchronize(st));
    plan->rounds = static_cast<int>(r + 1);
    if (!changed) break;
  }
  const long long nsub_chunks = (plan->nsub + SCAN_CHUNK - 1) / SCAN_CHUNK;
  jpeg_count_scan_local_kernel<<<static_cast<unsigned>(nsub_chunks), SCAN_CHUNK, 0, st>>>(p);
  int rc = post_launch("ovg_jpeg_decode(count scan)");
  if (rc) return rc;
  jpeg_count_scan_chunks_kernel<<<1, SCAN_CHUNK, 0, st>>>(w.chunk, nsub_chunks);
  if ((rc = post_launch("ovg_jpeg_decode(count scan chunks)"))) return rc;
  OVG_CUDA(cudaMemsetAsync(w.coef, 0, 128 * plan->nblocks, st));
  jpeg_write_kernel<<<sub_grid, 256, 0, st>>>(p);
  if ((rc = post_launch("ovg_jpeg_decode(write)"))) return rc;
  const long long nblk_chunks = (plan->nblocks + SCAN_CHUNK - 1) / SCAN_CHUNK;
  jpeg_dc_local_kernel<<<static_cast<unsigned>(nblk_chunks), SCAN_CHUNK, 0, st>>>(p);
  if ((rc = post_launch("ovg_jpeg_decode(dc scan)"))) return rc;
  jpeg_dc_chunks_kernel<<<1, SCAN_CHUNK, 0, st>>>(w.dc_agg, w.dc_aggf, nblk_chunks);
  if ((rc = post_launch("ovg_jpeg_decode(dc scan chunks)"))) return rc;
  jpeg_idct_kernel<<<static_cast<unsigned>((plan->nblocks + 127) / 128), 128, 0, st>>>(p);
  if ((rc = post_launch("ovg_jpeg_decode(idct)"))) return rc;
  jpeg_color_kernel<<<static_cast<unsigned>((plan->npix + 255) / 256), 256, 0, st>>>(p);
  return post_launch("ovg_jpeg_decode(color)");
}

}  // extern "C"

#include "runtime.inc"
