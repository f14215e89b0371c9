// libovg C ABI (include/ovg.h): argument validation, TMA descriptor cache, kernel launches.
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdlib>
#include <mutex>
#include <string>
#include <unordered_map>
#include <vector>

#include <cudaTypedefs.h>

#include "../../include/ovg.h"
#include "arena.cuh"
#include "attn.cuh"
#include "camera.cuh"
#include "elem.cuh"
#include "gemm.cuh"
#include "post.cuh"
#include "match.cuh"
#include "tracks.cuh"
#include "ba.cuh"
#include "mesh.cuh"
#include "tsdf.cuh"
#include "sky.cuh"
#include "fps.cuh"
#include "rank.cuh"
#include "sim3.cuh"
#include "eval.cuh"
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

// ------------------------------------------------------------------------------ workspaces
// Every component with a size query has one layout function, Bufs layout(Arena&, dims...).  Its size query answers
// layout_bytes(layout, dims...) and its entry points take their buffers from carve(), so the two cannot disagree.
using ovg::Arena;

template <typename Bufs, typename... P, typename... A>
long long layout_bytes(Bufs (*layout)(Arena&, P...), A... dims) {
  Arena ar(nullptr);
  layout(ar, dims...);
  return ar.bytes();
}

// The caller's workspace, checked to be non-null, Align-byte aligned and layout_bytes() long, carved into *out.  A failure
// names the entry point fn and the size query to call.
template <uintptr_t Align = 256, typename Bufs, typename... P, typename... A>
int carve(const char* fn, const char* query, const void* workspace, long long workspace_bytes, Bufs* out,
          Bufs (*layout)(Arena&, P...), A... dims) {
  if (!workspace || (reinterpret_cast<uintptr_t>(workspace) & (Align - 1)) != 0 ||
      workspace_bytes < layout_bytes(layout, dims...))
    return fail(OVG_E_INVALID, std::string(fn) + ": workspace must be " + std::to_string(Align) + "-byte aligned and " +
                                   query + " long");
  Arena ar(const_cast<void*>(workspace));
  *out = layout(ar, dims...);
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

int ovg_version(void) { return 5; }
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
    case OVG_EPI_QKV:   // bn is 64 or 128 (raised above)
      return bn == 128 ? launch_gemm<128, ovg::EPI_QKV>(ta, tb, p, st) : launch_gemm<64, ovg::EPI_QKV>(ta, tb, p, st);
    case OVG_EPI_HEADTAIL: return launch_gemm<32, ovg::EPI_HEADTAIL>(ta, tb, p, st);
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

// in_mode: ovg::LN_IN_F32, LN_IN_BF16 or LN_IN_F32_AS_BF16 (the last is internal: ovg_dpt_forward reads fp32 slots with it)
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

// layer: fp32 [K*T, 2C] export of the same half (ovg_aggregator_forward's layers), or NULL
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

// The percentile's workspace of OVG_PERCENTILE_WORKSPACE_BYTES, packed (not carved at 256-byte boundaries):
// 6 x u64 state | 512 x u32 histograms | 3 x f32 results | u32 NaN count.
struct PercentileRegion {
  unsigned long long* state;
  unsigned int* hist;
  float* res;
  unsigned int* nan;
};

PercentileRegion percentile_region(void* workspace) {
  unsigned long long* state = static_cast<unsigned long long*>(workspace);
  unsigned int* hist = reinterpret_cast<unsigned int*>(state + 6);
  float* res = reinterpret_cast<float*>(hist + 512);
  return {state, hist, res, reinterpret_cast<unsigned int*>(res + 3)};
}

// The 4 x (histogram, decide) passes of a radix selection whose ranks an init launch has set in the workspace's state.
// nan: the region's NaN counter for a percentile (see ovg::SelectParams), or null for a bare selection.
int radix_select_passes(const float* v, long long n, void* workspace, float* out3, unsigned int* nan, const std::string& what,
                        cudaStream_t st) {
  const PercentileRegion r = percentile_region(workspace);
  int rc = OVG_OK;
  const int blocks = select_blocks(n);
  for (int pass = 0; pass < 4; ++pass) {
    ovg::SelectParams sp{v, n, r.state, r.hist, pass, out3, nan};
    ovg::select_hist_kernel<<<blocks, 256, 0, st>>>(sp);
    rc = post_launch((what + "(hist)").c_str());
    if (rc) return rc;
    ovg::select_decide_kernel<<<1, 32, 0, st>>>(sp);
    rc = post_launch((what + "(decide)").c_str());
    if (rc) return rc;
  }
  return OVG_OK;
}

// numpy.percentile(v[0, n), percent) (method "linear", numpy >= 2's fp32 rule, exact) by radix select: one init launch that
// takes the ranks and weight on the device, then 4 x (histogram, decide).  workspace: a percentile_region; out3: device
// float[3] = the two neighbouring order statistics and the interpolated percentile, NaN if any v is NaN.  count (optional)
// is zeroed by the init launch.
int radix_percentile(const float* v, long long n, float percent, void* workspace, float* out3, unsigned long long* count,
                     const std::string& what, cudaStream_t st) {
  const PercentileRegion r = percentile_region(workspace);
  ovg::select_init_kernel<<<1, 128, 0, st>>>(r.state, r.hist, n, percent, out3 + 2, r.nan, count);
  const int rc = post_launch((what + "(init)").c_str());
  return rc ? rc : radix_select_passes(v, n, workspace, out3, r.nan, what, st);
}

struct CloudBufs {
  void* select;                      // OVG_PERCENTILE_WORKSPACE_BYTES
  float* sel;                        // [6][3] selection results of the scale
  double* center_partial;            // [CLOUD_CENTER_BLOCKS][3]
  unsigned int* tile_count;          // [tiles]
  unsigned long long* tile_offset;   // [tiles]
};

CloudBufs cloud_layout(Arena& ar, long long n) {
  CloudBufs w;
  w.select = ar.take(OVG_PERCENTILE_WORKSPACE_BYTES);
  w.sel = ar.get<float>(18);
  w.center_partial = ar.get<double>(3LL * ovg::CLOUD_CENTER_BLOCKS);
  w.tile_count = ar.get<unsigned int>(ovg::compact_tiles(n));
  w.tile_offset = ar.get<unsigned long long>(ovg::compact_tiles(n));
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
  float* res = percentile_region(workspace).res;
  int rc = radix_percentile(conf, n, percent, workspace, res, count_out, "ovg_conf_percentile_mask", st);
  if (rc) return rc;
  const int blocks = select_blocks(n);
  OVG_CUDA(cudaMemcpyAsync(threshold_out, res + 2, sizeof(float), cudaMemcpyDeviceToDevice, st));
  ovg::ConfMaskParams mp{conf, res + 2, mask, n, floor_, count_out};
  ovg::conf_mask_kernel<<<blocks, 256, 0, st>>>(mp);
  return post_launch("ovg_conf_percentile_mask");
}

long long ovg_point_cloud_workspace_bytes(long long n) { return n > 0 ? layout_bytes(cloud_layout, n) : -1; }

}  // extern "C"

namespace {

int cloud_params(const char* fn, const unsigned char* conf_mask, const float* images, int F, int H, int W, int mask_black_bg,
                 int mask_white_bg, const void* workspace, long long workspace_bytes, ovg::CloudParams* p) {
  OVG_REQUIRE(conf_mask && images && F > 0 && H > 0 && W > 0, "bad arguments");
  const long long n = static_cast<long long>(F) * H * W;
  CloudBufs w;
  const int rc = carve<16>(fn, "ovg_point_cloud_workspace_bytes(F*H*W)", workspace, workspace_bytes, &w, cloud_layout, n);
  if (rc) return rc;
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
  int rc = cloud_params(__func__, conf_mask, images, F, H, W, mask_black_bg, mask_white_bg, workspace, workspace_bytes, &p);
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
  int rc = cloud_params(__func__, conf_mask, images, F, H, W, mask_black_bg, mask_white_bg, workspace, workspace_bytes, &p);
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
  OVG_REQUIRE(points && center_out && n > 0, "bad arguments");
  CloudBufs w;
  int rc = carve<16>(__func__, "ovg_point_cloud_workspace_bytes(n)", workspace, workspace_bytes, &w, cloud_layout, n);
  if (rc) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ovg::CloudCenterParams p{points, n, w.center_partial, center_out};
  ovg::cloud_center_partial_kernel<<<ovg::CLOUD_CENTER_BLOCKS, 256, 0, st>>>(p);
  rc = post_launch("ovg_point_cloud_center");
  if (rc) return rc;
  ovg::cloud_center_final_kernel<<<1, 32, 0, st>>>(p);
  return post_launch("ovg_point_cloud_center(final)");
}

int ovg_point_cloud_scale(const float* xyz, long long n_kept, long long ld, void* workspace, long long workspace_bytes,
                          float* scale_out, void* stream) {
  OVG_REQUIRE(xyz && scale_out && n_kept > 0 && ld >= n_kept && ld % 4 == 0, "bad arguments");
  OVG_REQUIRE((reinterpret_cast<uintptr_t>(xyz) & 15) == 0, "xyz must be 16-byte aligned");
  CloudBufs w;     // the scale uses only the fixed-size head of the workspace: the layout of one point
  int rc = carve<16>(__func__, "ovg_point_cloud_workspace_bytes()", workspace, workspace_bytes, &w, cloud_layout, 1LL);
  if (rc) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  for (int q = 0; q < 2; ++q)
    for (int a = 0; a < 3; ++a) {
      rc = radix_percentile(xyz + a * ld, n_kept, q ? 95.f : 5.f, w.select, w.sel + (q * 3 + a) * 3, nullptr,
                            "ovg_point_cloud_scale", st);
      if (rc) return rc;
    }
  ovg::cloud_scale_kernel<<<1, 32, 0, st>>>(w.sel, scale_out);
  return post_launch("ovg_point_cloud_scale");
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------- reciprocal matches
namespace {

struct MatchBufs {
  ovg::MatchParams p;
  int passes;          // 8-bit radix-sort passes over the cell ids
};

MatchBufs match_layout(Arena& ar, int V, long long cap, int P) {
  MatchBufs w;
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
  return w;
}

int match_check(const char* fn, int V, long long cap, int P, const void* workspace, long long workspace_bytes,
                ovg::MatchParams* p, int* passes = nullptr) {
  // cap < 2^30 keeps the cell ids (cells_cap = 2 cap + 64) and the slots inside a view in int range
  OVG_REQUIRE(V > 0 && V <= 65535 && cap > 0 && cap < (1LL << 30) && P > 0 && 2LL * P <= 65535, "bad sizes");
  OVG_REQUIRE(static_cast<long long>(V) * cap < (1LL << 40), "too many points");
  MatchBufs w;
  const int rc = carve(fn, "ovg_match_workspace_bytes(V, cap, P)", workspace, workspace_bytes, &w, match_layout, V, cap, P);
  if (rc) return rc;
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
  return (V > 0 && cap > 0 && P > 0) ? layout_bytes(match_layout, V, cap, P) : -1;
}

int ovg_match_index(const float* points, const unsigned char* keep, int V, long long cap, int P, void* workspace,
                    long long workspace_bytes, void* stream) {
  ovg::MatchParams p;
  int passes = 0;
  int rc = match_check(__func__, V, cap, P, workspace, workspace_bytes, &p, &passes);
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
  int rc = match_check(__func__, V, cap, P, workspace, workspace_bytes, &p);
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
  int rc = match_check(__func__, V, cap, P, workspace, workspace_bytes, &p);
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
  int rc = match_check(__func__, V, cap, P, workspace, workspace_bytes, &p);
  if (rc) return rc;
  OVG_REQUIRE(pairs && reciprocal && nn && pair >= 0 && pair < P, "bad arguments");
  p.pairs = pairs;
  ovg::MatchOut o{1, nullptr, nullptr, pair, reciprocal, nn};
  ovg::match_pair_kernel<<<static_cast<unsigned>((cap + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p, o);
  return post_launch("ovg_match_pair");
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------- star tracks
namespace {

ovg::TrackParams tracks_layout(Arena& ar, int V, long long cap) {
  ovg::TrackParams p{};
  const long long nodes = V * cap;
  const long long tiles = ovg::compact_tiles(cap) * (V > 2 ? V : 2);
  p.claim = ar.get<int>(nodes);
  p.rank = ar.get<int>(nodes);
  p.obs = ar.get<int>(nodes);
  p.track_start = ar.get<int>(nodes);
  p.tile_count = ar.get<unsigned int>(tiles);
  p.tile_offset = ar.get<unsigned long long>(tiles);
  p.scan_total = ar.get<unsigned long long>(1);
  p.totals = ar.get<unsigned long long>(4);
  return p;
}

int tracks_check(const char* fn, int V, long long cap, int P, const void* match_ws, long long match_ws_bytes, void* workspace,
                 long long workspace_bytes, ovg::TrackParams* p) {
  OVG_REQUIRE(V > 0 && cap > 0 && static_cast<long long>(V) * cap < (1LL << 31), "V * cap must be below 2^31");
  ovg::MatchParams m;
  int rc = match_check(fn, V, cap, P, match_ws, match_ws_bytes, &m);
  if (rc) return rc;
  rc = carve(fn, "ovg_tracks_workspace_bytes(V, cap)", workspace, workspace_bytes, p, tracks_layout, V, cap);
  p->m = m;
  return rc;
}

}  // namespace

extern "C" {

long long ovg_tracks_workspace_bytes(int V, long long cap) {
  return (V > 0 && cap > 0) ? layout_bytes(tracks_layout, V, cap) : -1;
}

int ovg_tracks_assign(const int* pairs, const int* pair_off, int P, int V, long long cap, int min_views, const void* match_workspace,
                      long long match_workspace_bytes, void* workspace, long long workspace_bytes, long long* counts_out,
                      void* stream) {
  ovg::TrackParams p{};
  int rc = tracks_check(__func__, V, cap, P, match_workspace, match_workspace_bytes, workspace, workspace_bytes, &p);
  if (rc) return rc;
  OVG_REQUIRE(pairs && pair_off && counts_out, "null pairs / pair_off / counts_out");
  OVG_REQUIRE(min_views >= 1 && min_views <= V, "min_views must be in [1, V]");
  p.m.pairs = pairs;
  p.pair_off = pair_off;
  p.min_views = min_views;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  OVG_CUDA(cudaMemsetAsync(p.claim, 0xFF, 4LL * V * cap, st));
  OVG_CUDA(cudaMemsetAsync(p.totals, 0, 2 * sizeof(unsigned long long), st));
  const int tiles = p.m.tiles;
  for (int a = 0; a < V; ++a) {
    ovg::track_count_kernel<<<tiles, ovg::COMPACT_THREADS, 0, st>>>(p, a);
    if ((rc = post_launch("ovg_tracks_assign(count)"))) return rc;
    ovg::tile_scan_kernel<<<1, 1024, 0, st>>>(p.tile_count, p.tile_offset, p.scan_total, 2LL * tiles);
    if ((rc = post_launch("ovg_tracks_assign(scan)"))) return rc;
    ovg::track_write_kernel<<<tiles, ovg::COMPACT_THREADS, 0, st>>>(p, a);
    if ((rc = post_launch("ovg_tracks_assign(write)"))) return rc;
  }
  ovg::track_counts_kernel<<<1, 1, 0, st>>>(p, counts_out);
  return post_launch("ovg_tracks_assign(counts)");
}

int ovg_tracks_gather(const float* images, const float* extrinsic, const float* intrinsic, int V, long long cap, int P, int W,
                      long long n_tracks, long long n_obs, const void* match_workspace, long long match_workspace_bytes,
                      void* workspace, long long workspace_bytes, double* points, unsigned char* colors, double* error,
                      long long* offsets, int* view, long long* xy, int* point2d, long long* view_offsets, int* view_track,
                      long long* view_xy, void* stream) {
  ovg::TrackParams p{};
  int rc = tracks_check(__func__, V, cap, P, match_workspace, match_workspace_bytes, workspace, workspace_bytes, &p);
  if (rc) return rc;
  OVG_REQUIRE(W > 0 && cap % W == 0, "cap must be H * W");
  OVG_REQUIRE(n_tracks >= 0 && n_tracks <= n_obs && n_obs <= static_cast<long long>(V) * cap, "bad track counts");
  OVG_REQUIRE(offsets && view_offsets, "null offsets / view_offsets");
  OVG_REQUIRE(n_tracks == 0 || (images && extrinsic && intrinsic && points && colors && error && view && xy && point2d &&
                                view_track && view_xy), "null operand");
  const ovg::TrackOut o{images, extrinsic, intrinsic, W, n_tracks, n_obs, points, colors, error, offsets, view, xy, point2d,
                        view_offsets, view_track, view_xy};
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const dim3 grid(p.m.tiles, V);
  ovg::track_claimed_kernel<<<grid, ovg::COMPACT_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_tracks_gather(claimed count)"))) return rc;
  ovg::tile_scan_kernel<<<1, 1024, 0, st>>>(p.tile_count, p.tile_offset, p.scan_total, static_cast<long long>(V) * p.m.tiles);
  if ((rc = post_launch("ovg_tracks_gather(scan)"))) return rc;
  ovg::track_view_kernel<<<grid, ovg::COMPACT_THREADS, 0, st>>>(p, o);
  if ((rc = post_launch("ovg_tracks_gather(views)"))) return rc;
  if (n_tracks == 0) {
    OVG_CUDA(cudaMemsetAsync(offsets, 0, sizeof(long long), st));
    return OVG_OK;
  }
  ovg::track_point_kernel<<<static_cast<unsigned>((n_tracks + ovg::TRACK_POINT_THREADS - 1) / ovg::TRACK_POINT_THREADS),
                            ovg::TRACK_POINT_THREADS, 0, st>>>(p, o);
  return post_launch("ovg_tracks_gather(points)");
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------- bundle adjustment
namespace {

ovg::BaParams ba_layout(Arena& ar, int V, long long n, long long m) {
  ovg::BaParams p{};
  p.tblocks = static_cast<int>(std::max(1LL, (n + ovg::BA_THREADS - 1) / ovg::BA_THREADS));
  p.vtiles = static_cast<int>(std::max(1LL, ovg::compact_tiles(m)));
  p.st = ar.get<ovg::BaState>(1);
  p.cam = ar.get<double>(2LL * V * ovg::BA_CAM);
  p.mask = ar.get<double>(static_cast<long long>(V) * ovg::BA_NP);
  p.dcam = ar.get<double>(static_cast<long long>(V) * ovg::BA_NP);
  p.pts = ar.get<double>(6 * n);
  p.dp = ar.get<double>(3 * n);
  p.vinv = ar.get<double>(9 * n);
  p.y = ar.get<double>(3 * n);
  p.gp = ar.get<double>(3 * n);
  p.zt = ar.get<double>(3 * n);
  p.incl = ar.get<unsigned char>(n);
  p.ob = ar.get<ovg::BaObs>(m);
  p.obs_track = ar.get<int>(m);
  p.view_obs = ar.get<int>(m);
  p.view_off = ar.get<long long>(V + 1);
  p.gmax = ar.get<double>(p.tblocks);
  p.vpart = ar.get<double>(static_cast<long long>(V) * ovg::BA_BLOCK_CHUNKS * ovg::BA_ENTRIES);
  p.vsum = ar.get<double>(static_cast<long long>(V) * ovg::BA_ENTRIES);
  p.bpart = ar.get<double>(static_cast<long long>(V) * ovg::BA_PCG_CHUNKS * ovg::BA_NP);
  p.epart = ar.get<double>(static_cast<long long>(p.tblocks) * ovg::BA_EVAL);
  p.tile_count = ar.get<unsigned int>(static_cast<long long>(V) * p.vtiles);
  p.tile_offset = ar.get<unsigned long long>(static_cast<long long>(V) * p.vtiles);
  p.scan_total = ar.get<unsigned long long>(1);
  return p;
}

bool ba_sizes_ok(int V, long long n, long long m) {
  return V >= 2 && V <= ovg::BA_MAX_VIEWS && n >= 0 && m >= 0 && n < (1LL << 31) && m < (1LL << 31);
}

}  // namespace

extern "C" {

long long ovg_ba_workspace_bytes(int V, long long n_tracks, long long n_obs) {
  return ba_sizes_ok(V, n_tracks, n_obs) ? layout_bytes(ba_layout, V, n_tracks, n_obs) : -1;
}

int ovg_bundle_adjust(const double* points, const long long* offsets, const int* view, const double* observations,
                      const float* extrinsic, const float* intrinsic, int V, long long n_tracks, long long n_obs, int iterations,
                      int refine_focal, int loss, double loss_scale, void* workspace, long long workspace_bytes,
                      double* points_out, double* extrinsic_out, double* intrinsic_out, double* error_out, double* cost_out,
                      long long* stats_out, double* trace_out, void* stream) {
  OVG_REQUIRE(ba_sizes_ok(V, n_tracks, n_obs), "need 2 <= V <= 256 and 0 <= n_tracks, n_obs < 2^31");
  OVG_REQUIRE(iterations >= 1, "iterations must be >= 1");
  OVG_REQUIRE(loss == OVG_BA_LOSS_TRIVIAL || loss == OVG_BA_LOSS_CAUCHY, "unknown loss");
  OVG_REQUIRE(std::isfinite(loss_scale) && loss_scale > 0.0, "loss_scale must be finite and > 0");
  OVG_REQUIRE(offsets && extrinsic && intrinsic && extrinsic_out && intrinsic_out && cost_out && stats_out, "null operand");
  OVG_REQUIRE(n_tracks == 0 || (points && points_out && error_out), "null points / points_out / error_out");
  OVG_REQUIRE(n_obs == 0 || (view && observations), "null view / observations");
  ovg::BaParams p;
  int rc = carve(__func__, "ovg_ba_workspace_bytes(V, n_tracks, n_obs)", workspace, workspace_bytes, &p, ba_layout, V, n_tracks,
                 n_obs);
  if (rc) return rc;
  p.V = V; p.n = n_tracks; p.m = n_obs; p.iterations = iterations; p.refine_focal = refine_focal ? 1 : 0;
  p.cauchy = loss == OVG_BA_LOSS_CAUCHY; p.c2 = loss_scale * loss_scale;
  p.points = points; p.offsets = offsets; p.view = view; p.obs = observations; p.ext = extrinsic; p.intr = intrinsic;
  p.points_out = points_out; p.ext_out = extrinsic_out; p.intr_out = intrinsic_out; p.error_out = error_out;
  p.cost_out = cost_out; p.stats_out = stats_out; p.trace = trace_out;
  // the PCG spins on the other CTAs: launched cooperatively with the grid the occupancy query allows
  const int smem = ovg::BA_VIEW_SMEM * V * static_cast<int>(sizeof(double));
  rc = allow_dynamic_smem<ovg::ba_pcg_kernel>(ovg::BA_VIEW_SMEM * ovg::BA_MAX_VIEWS * static_cast<int>(sizeof(double)));
  if (rc) return rc;
  int per_sm = 0;
  OVG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ovg::ba_pcg_kernel, ovg::BA_PCG_THREADS, smem));
  OVG_REQUIRE(per_sm > 0, "the PCG kernel does not fit on an SM");
  const int grid = per_sm * num_sms();
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const unsigned tb = static_cast<unsigned>(p.tblocks);
  const dim3 vgrid(p.vtiles, V);
  ovg::ba_init_kernel<<<1, 1, 0, st>>>(p);
  if ((rc = post_launch("ovg_bundle_adjust(init)"))) return rc;
  ovg::ba_track_init_kernel<<<tb, ovg::BA_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_bundle_adjust(track init)"))) return rc;
  ovg::ba_view_count_kernel<<<vgrid, ovg::COMPACT_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_bundle_adjust(view count)"))) return rc;
  ovg::tile_scan_kernel<<<1, 1024, 0, st>>>(p.tile_count, p.tile_offset, p.scan_total, static_cast<long long>(V) * p.vtiles);
  if ((rc = post_launch("ovg_bundle_adjust(scan)"))) return rc;
  ovg::ba_view_gather_kernel<<<vgrid, ovg::COMPACT_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_bundle_adjust(view gather)"))) return rc;
  ovg::ba_eval_kernel<<<tb, ovg::BA_THREADS, 0, st>>>(p, 0);
  if ((rc = post_launch("ovg_bundle_adjust(initial cost)"))) return rc;
  ovg::ba_control_kernel<<<1, ovg::BA_PCG_THREADS, 0, st>>>(p, 1);
  if ((rc = post_launch("ovg_bundle_adjust(initial control)"))) return rc;
  void* args[] = {&p};
  for (int i = 0; i < iterations; ++i) {                     // after a stop every kernel returns at once
    ovg::ba_track_kernel<<<tb, ovg::BA_THREADS, 0, st>>>(p);
    if ((rc = post_launch("ovg_bundle_adjust(tracks)"))) return rc;
    ovg::ba_view_block_kernel<<<dim3(ovg::BA_BLOCK_CHUNKS, V), ovg::BA_BLOCK_THREADS, 0, st>>>(p);
    if ((rc = post_launch("ovg_bundle_adjust(view blocks)"))) return rc;
    ovg::ba_view_reduce_kernel<<<V, ovg::BA_BLOCK_THREADS, 0, st>>>(p);
    if ((rc = post_launch("ovg_bundle_adjust(view sums)"))) return rc;
    OVG_CUDA(cudaLaunchCooperativeKernel(reinterpret_cast<void*>(ovg::ba_pcg_kernel), dim3(grid), dim3(ovg::BA_PCG_THREADS),
                                         args, smem, st));
    if ((rc = post_launch("ovg_bundle_adjust(pcg)"))) return rc;
    ovg::ba_eval_kernel<<<tb, ovg::BA_THREADS, 0, st>>>(p, 1);
    if ((rc = post_launch("ovg_bundle_adjust(trial cost)"))) return rc;
    ovg::ba_control_kernel<<<1, ovg::BA_PCG_THREADS, 0, st>>>(p, 0);
    if ((rc = post_launch("ovg_bundle_adjust(control)"))) return rc;
  }
  ovg::ba_output_kernel<<<tb, ovg::BA_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_bundle_adjust(points)"))) return rc;
  ovg::ba_finish_kernel<<<1, 32, 0, st>>>(p);
  return post_launch("ovg_bundle_adjust(finish)");
}

}  // extern "C"

// -------------------------------------------------------------------------------------------------------------- triangle mesh
namespace {

ovg::MeshParams mesh_layout(Arena& ar, int F, int H, int W) {
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
  return p;
}

int mesh_check(const char* fn, int F, int H, int W, const void* workspace, long long workspace_bytes, ovg::MeshParams* p) {
  OVG_REQUIRE(F > 0 && F <= 65535 && H > 0 && W > 0, "bad sizes");
  OVG_REQUIRE(static_cast<long long>(F) * H * W < (1LL << 31), "F*H*W must be below 2^31");
  return carve(fn, "ovg_mesh_workspace_bytes(F, H, W)", workspace, workspace_bytes, p, mesh_layout, F, H, W);
}

}  // namespace

extern "C" {

long long ovg_mesh_workspace_bytes(int F, int H, int W) {
  return (F > 0 && H > 0 && W > 0) ? layout_bytes(mesh_layout, F, H, W) : -1;
}

int ovg_mesh_count(const unsigned char* conf_mask, const float* images, int F, int H, int W, int mask_black_bg,
                   int mask_white_bg, void* workspace, long long workspace_bytes, long long* counts_out, void* stream) {
  ovg::MeshParams p;
  int rc = mesh_check(__func__, F, H, W, workspace, workspace_bytes, &p);
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
  int rc = mesh_check(__func__, F, H, W, workspace, workspace_bytes, &p);
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
  int rc = mesh_check(__func__, F, H, W, workspace, workspace_bytes, &p);
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

// -------------------------------------------------------------------------------------------------------------- fused mesh
namespace {

// The TSDF workspace holds two parts, each carved from its start: the bounds part of F*H*W points and the volume part of an
// nx x ny x nz grid.  ovg_tsdf_workspace_bytes is the larger of the two.
struct TsdfBoundsBufs {
  void* select;                      // OVG_PERCENTILE_WORKSPACE_BYTES
  float* sel;                        // [6][3] selection results, in the order (axis, percentile)
  float* frac;                       // [6] their interpolation weights
  unsigned long long* count;
  unsigned int* nonfinite;
  float* cols;                       // [3, ld]
  long long ld;
};

TsdfBoundsBufs tsdf_bounds_layout(Arena& ar, long long n) {
  TsdfBoundsBufs w;
  w.ld = (n + 3) / 4 * 4;
  w.select = ar.take(OVG_PERCENTILE_WORKSPACE_BYTES);
  w.sel = ar.get<float>(18);
  w.frac = ar.get<float>(6);
  w.count = ar.get<unsigned long long>(1);
  w.nonfinite = ar.get<unsigned int>(1);
  w.cols = ar.get<float>(3 * w.ld);
  return w;
}

struct TsdfVolumeBufs {
  unsigned char* marked;             // [bricks]
  unsigned int* tile_count;          // [2 bricks]
  unsigned long long* tile_offset;   // [2 bricks + 1]
  int* edge_vertex;                  // [nz, ny, nx, 3]
  long long bricks;
};

TsdfVolumeBufs tsdf_volume_layout(Arena& ar, int nx, int ny, int nz) {
  TsdfVolumeBufs w;
  w.bricks = static_cast<long long>((nx + 7) / 8) * ((ny + 7) / 8) * ((nz + 7) / 8);
  w.marked = ar.get<unsigned char>(w.bricks);
  w.tile_count = ar.get<unsigned int>(2 * w.bricks);
  w.tile_offset = ar.get<unsigned long long>(2 * w.bricks + 1);
  w.edge_vertex = ar.get<int>(3LL * nx * ny * nz);
  return w;
}

bool tsdf_triple(int a, int b, int c) { return (a > 0 && b > 0 && c > 0) || (a == 0 && b == 0 && c == 0); }

int tsdf_grid(const char* fn, int nx, int ny, int nz, float ox, float oy, float oz, float voxel, float trunc,
              const void* workspace, long long workspace_bytes, TsdfVolumeBufs* w, ovg::TsdfGrid* g) {
  OVG_REQUIRE(nx > 0 && ny > 0 && nz > 0 && 3LL * nx * ny * nz < (1LL << 31), "need 0 < nx, ny, nz and 3 nx ny nz < 2^31");
  OVG_REQUIRE(std::isfinite(ox) && std::isfinite(oy) && std::isfinite(oz) && std::isfinite(voxel) && voxel > 0.f &&
                  std::isfinite(trunc) && trunc > 0.f,
              "origin, voxel and trunc must be finite, voxel and trunc > 0");
  *g = ovg::TsdfGrid{nx, ny, nz, (nx + 7) / 8, (ny + 7) / 8, (nz + 7) / 8, ox, oy, oz, voxel, trunc};
  return carve(fn, "ovg_tsdf_workspace_bytes(nx, ny, nz, ...)", workspace, workspace_bytes, w, tsdf_volume_layout, nx, ny, nz);
}

int tsdf_mesh(const char* fn, const float* tsdf, int nx, int ny, int nz, float ox, float oy, float oz, float voxel,
              const void* workspace, long long workspace_bytes, ovg::TsdfMeshParams* p) {
  OVG_REQUIRE(tsdf, "null tsdf");
  TsdfVolumeBufs w;
  *p = ovg::TsdfMeshParams{};
  const int rc = tsdf_grid(fn, nx, ny, nz, ox, oy, oz, voxel, 1.f, workspace, workspace_bytes, &w, &p->g);
  if (rc) return rc;
  p->tsdf = tsdf; p->bricks = w.bricks;
  p->tile_count = w.tile_count; p->tile_offset = w.tile_offset; p->edge_vertex = w.edge_vertex;
  return OVG_OK;
}

}  // namespace

extern "C" {

long long ovg_tsdf_workspace_bytes(int nx, int ny, int nz, int F, int H, int W) {
  if (!tsdf_triple(nx, ny, nz) || !tsdf_triple(F, H, W) || (nx == 0 && F == 0)) return -1;
  if (3LL * nx * ny * nz >= (1LL << 31) || static_cast<long long>(F) * H * W >= (1LL << 31)) return -1;
  return std::max(F ? layout_bytes(tsdf_bounds_layout, static_cast<long long>(F) * H * W) : 0LL,
                  nx ? layout_bytes(tsdf_volume_layout, nx, ny, nz) : 0LL);
}

int ovg_tsdf_bounds(const float* points, const unsigned char* mask, int F, int H, int W, void* workspace,
                    long long workspace_bytes, double* bounds_out, void* stream) {
  OVG_REQUIRE(points && mask && bounds_out, "null operand");
  OVG_REQUIRE(F > 0 && H > 0 && W > 0 && static_cast<long long>(F) * H * W < (1LL << 31), "need F H W < 2^31");
  const long long n = static_cast<long long>(F) * H * W;
  TsdfBoundsBufs w;
  int rc = carve(__func__, "ovg_tsdf_workspace_bytes(..., F, H, W)", workspace, workspace_bytes, &w, tsdf_bounds_layout, n);
  if (rc) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  OVG_CUDA(cudaMemsetAsync(w.count, 0, sizeof(unsigned long long), st));
  OVG_CUDA(cudaMemsetAsync(w.nonfinite, 0, sizeof(unsigned int), st));
  const ovg::TsdfBoundsParams bp{points, mask, n, w.ld, w.cols, w.count, w.nonfinite};
  ovg::tsdf_fill_kernel<<<select_blocks(n), 256, 0, st>>>(bp);
  rc = post_launch("ovg_tsdf_bounds(fill)");
  if (rc) return rc;
  const PercentileRegion r = percentile_region(w.select);
  for (int j = 0; j < 6; ++j) {          // j = 2 axis + (0: 1st percentile, 1: 99th)
    ovg::tsdf_select_init_kernel<<<1, 128, 0, st>>>(r.state, r.hist, w.count, (j & 1) ? 99.f : 1.f, w.frac + j);
    if ((rc = post_launch("ovg_tsdf_bounds(init)"))) return rc;
    // a bare selection: tsdf_bounds_kernel weighs the pair with the device's frac
    if ((rc = radix_select_passes(w.cols + (j >> 1) * w.ld, n, w.select, w.sel + 3 * j, nullptr, "ovg_tsdf_bounds", st)))
      return rc;
  }
  ovg::tsdf_bounds_kernel<<<1, 32, 0, st>>>(w.sel, w.frac, w.count, w.nonfinite, bounds_out);
  return post_launch("ovg_tsdf_bounds");
}

int ovg_tsdf_integrate(const float* depth, const unsigned char* mask, const float* images, const float* extrinsic,
                       const float* intrinsic, int F, int H, int W, int nx, int ny, int nz, float ox, float oy, float oz,
                       float voxel, float trunc, void* workspace, long long workspace_bytes, float* tsdf, unsigned char* color,
                       void* stream) {
  OVG_REQUIRE(depth && mask && images && extrinsic && intrinsic && tsdf && color, "null operand");
  OVG_REQUIRE(F > 0 && H > 0 && W > 0 && static_cast<long long>(F) * H * W < (1LL << 31), "need F H W < 2^31");
  TsdfVolumeBufs w;
  ovg::TsdfIntegrateParams p{};
  int rc = tsdf_grid(__func__, nx, ny, nz, ox, oy, oz, voxel, trunc, workspace, workspace_bytes, &w, &p.g);
  if (rc) return rc;
  OVG_REQUIRE((reinterpret_cast<uintptr_t>(color) & 3) == 0, "color must be 4-byte aligned");
  p.depth = depth; p.mask = mask; p.images = images; p.ext = extrinsic; p.intr = intrinsic;
  p.F = F; p.H = H; p.W = W;
  p.marked = w.marked; p.tsdf = tsdf; p.color = color;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  OVG_CUDA(cudaMemsetAsync(w.marked, 0, w.bricks, st));
  const long long n = static_cast<long long>(F) * H * W;
  ovg::tsdf_mark_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(p);
  if ((rc = post_launch("ovg_tsdf_integrate(mark)"))) return rc;
  ovg::tsdf_integrate_kernel<<<static_cast<unsigned>(w.bricks), ovg::TSDF_BRICK_VOXELS, 0, st>>>(p);
  return post_launch("ovg_tsdf_integrate");
}

int ovg_tsdf_count(const float* tsdf, int nx, int ny, int nz, void* workspace, long long workspace_bytes, long long* counts_out,
                   void* stream) {
  ovg::TsdfMeshParams p;
  int rc = tsdf_mesh(__func__, tsdf, nx, ny, nz, 0.f, 0.f, 0.f, 1.f, workspace, workspace_bytes, &p);
  if (rc) return rc;
  OVG_REQUIRE(counts_out, "null counts_out");
  p.totals = counts_out;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ovg::tsdf_count_kernel<<<static_cast<unsigned>(p.bricks), ovg::COMPACT_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_tsdf_count"))) return rc;
  ovg::tile_scan_kernel<<<1, 1024, 0, st>>>(p.tile_count, p.tile_offset, p.tile_offset + 2 * p.bricks, 2 * p.bricks);
  if ((rc = post_launch("ovg_tsdf_count(scan)"))) return rc;
  ovg::tsdf_totals_kernel<<<1, 32, 0, st>>>(p);
  return post_launch("ovg_tsdf_count(totals)");
}

int ovg_tsdf_extract(const float* tsdf, const unsigned char* color, int nx, int ny, int nz, float ox, float oy, float oz,
                     float voxel, void* workspace, long long workspace_bytes, float* positions, unsigned char* colors,
                     int* indices, void* stream) {
  ovg::TsdfMeshParams p;
  int rc = tsdf_mesh(__func__, tsdf, nx, ny, nz, ox, oy, oz, voxel, workspace, workspace_bytes, &p);
  if (rc) return rc;
  OVG_REQUIRE(color && positions && colors && indices, "null operand");
  p.color = color; p.positions = positions; p.colors = colors; p.indices = indices;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ovg::tsdf_vertices_kernel<<<static_cast<unsigned>(p.bricks), ovg::COMPACT_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_tsdf_extract(vertices)"))) return rc;
  ovg::tsdf_triangles_kernel<<<static_cast<unsigned>(p.bricks), ovg::COMPACT_THREADS, 0, st>>>(p);
  return post_launch("ovg_tsdf_extract(triangles)");
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------- sky segmentation
namespace {

ovg::SkyParams sky_layout(Arena& ar, int F, int H, int W) {
  ovg::SkyParams p{};
  p.F = F; p.H = H; p.W = W;
  p.hw = static_cast<long long>(H) * W;
  p.n = F * p.hw;
  p.tiles_x = (W + ovg::SKY_TILE - 1) / ovg::SKY_TILE;
  p.label = ar.get<int>(p.n);
  p.area = ar.get<int>(p.n);
  p.view_max = ar.get<int>(F);
  return p;
}

}  // namespace

extern "C" {

long long ovg_sky_workspace_bytes(int F, int H, int W) {
  return (F > 0 && H > 0 && W > 0) ? layout_bytes(sky_layout, F, H, W) : -1;
}

int ovg_segment_sky(const void* image, int image_u8, long long view_stride, long long pixel_stride, long long channel_stride,
                    int F, int H, int W, const float* conf, void* workspace, long long workspace_bytes, unsigned char* sky_out,
                    float* conf_out, void* stream) {
  OVG_REQUIRE(F > 0 && F <= 65535 && H > 0 && W > 0, "bad sizes");
  OVG_REQUIRE(static_cast<long long>(F) * H * W < (1LL << 31), "F*H*W must be below 2^31");
  OVG_REQUIRE(image && sky_out && (conf == nullptr) == (conf_out == nullptr), "null image / sky_out, or conf without conf_out");
  ovg::SkyParams p;
  int rc = carve(__func__, "ovg_sky_workspace_bytes(F, H, W)", workspace, workspace_bytes, &p, sky_layout, F, H, W);
  if (rc) return rc;
  p.image = image; p.u8 = image_u8 ? 1 : 0;
  p.view_stride = view_stride; p.pixel_stride = pixel_stride; p.channel_stride = channel_stride;
  p.conf = conf; p.conf_out = conf_out; p.sky = sky_out;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int tiles = p.tiles_x * ((H + ovg::SKY_TILE - 1) / ovg::SKY_TILE);
  ovg::sky_open_kernel<<<dim3(tiles, F), ovg::SKY_THREADS, 0, st>>>(p);
  rc = post_launch("ovg_segment_sky(colour test, opening)");
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

ovg::FpsParams fps_layout(Arena& ar, int B, long long N) {
  ovg::FpsParams p{};
  p.B = B; p.N = N;
  p.arrive = ar.get<unsigned>(B);
  p.slots = ar.get<ovg::FpsSlot>(2LL * ovg::FPS_MAX_CTAS);
  p.dist = ar.get<float>(static_cast<long long>(B) * N);
  return p;
}

}  // namespace

extern "C" {

long long ovg_fps_workspace_bytes(int B, long long N) {
  return (B > 0 && N > 0) ? layout_bytes(fps_layout, B, N) : -1;
}

int ovg_farthest_point_sample(const float* xyz, int B, long long N, int npoint, const long long* start, int include_ends,
                              void* workspace, long long workspace_bytes, long long* inds_out, void* stream) {
  OVG_REQUIRE(B > 0 && N > 0 && npoint > 0, "bad sizes");
  OVG_REQUIRE(N < (1LL << 31), "N must be below 2^31");
  OVG_REQUIRE(npoint <= N, "npoint must be <= N");
  OVG_REQUIRE(static_cast<long long>(B) * N < (1LL << 40), "too many points");
  OVG_REQUIRE(xyz && inds_out && (start || include_ends), "null xyz / inds_out, or no start without include_ends");
  ovg::FpsParams p;
  int rc = carve(__func__, "ovg_fps_workspace_bytes(B, N)", workspace, workspace_bytes, &p, fps_layout, B, N);
  if (rc) return rc;
  p.xyz = xyz; p.start = start; p.inds = inds_out; p.npoint = npoint; p.ends = include_ends ? 1 : 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (N <= ovg::FPS_CTA_POINTS) {   // one CTA per batch, every point in its shared memory
    rc = allow_dynamic_smem<ovg::fps_cta_kernel>(ovg::FPS_SMEM_BYTES);
    if (rc) return rc;
    ovg::fps_cta_kernel<<<B, ovg::FPS_THREADS, static_cast<int>(N) * 16, st>>>(p);
    return post_launch("ovg_farthest_point_sample(cta)");
  }
  // The grid kernel spins on the other CTAs of its group: launched cooperatively, sized by the occupancy query, so the
  // launch fails rather than run with CTAs that are not co-resident.
  rc = allow_dynamic_smem<ovg::fps_grid_kernel>(ovg::FPS_SMEM_BYTES);
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

// The packed operands, and on the grid path one scratch of two key / index buffers per CTA.
ovg::RankParams ranking_layout(Arena& ar, long long N, int out_f64) {
  ovg::RankParams p{};
  p.pose = ar.get<double>(N * 12);
  if (N > ovg::RANK_CTA_VIEWS) {
    p.scratch_stride = (N * (2 * (out_f64 ? 8 : 4) + 8) + 255) & ~255LL;
    p.scratch = ar.get<unsigned char>(ovg::RANK_GRID_CTAS * p.scratch_stride);
  }
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
  return (N > 0 && N < (1LL << 31)) ? layout_bytes(ranking_layout, N, out_f64) : -1;
}

int ovg_compute_ranking(const void* extrinsics, int in_f64, long long N, long long view_stride, long long row_stride,
                        long long col_stride, double lambda_t, int normalize, int out_f64, long long k, void* workspace,
                        long long workspace_bytes, long long* ranking, void* dists, void* stream) {
  OVG_REQUIRE(N > 0 && N < (1LL << 31), "N must be in [1, 2^31)");
  OVG_REQUIRE(k >= 1 && k <= N, "k must be in [1, N]");
  OVG_REQUIRE(extrinsics && ranking && dists, "null extrinsics / ranking / dists");
  ovg::RankParams p;
  int rc = carve(__func__, "ovg_ranking_workspace_bytes(N, out_f64)", workspace, workspace_bytes, &p, ranking_layout, N,
                 out_f64);
  if (rc) return rc;
  p.ext = extrinsics; p.s0 = view_stride; p.s1 = row_stride; p.s2 = col_stride;
  p.ranking = ranking; p.dists = dists; p.lambda = lambda_t;
  p.N = static_cast<int>(N); p.k = static_cast<int>(k);
  p.in_f64 = in_f64 ? 1 : 0; p.out_f64 = out_f64 ? 1 : 0; p.normalize = normalize ? 1 : 0;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ovg::rank_prep_kernel<<<1, ovg::RANK_PREP_THREADS, 0, st>>>(p);
  rc = post_launch("ovg_compute_ranking(prep)");
  if (rc) return rc;
  return p.out_f64 ? launch_ranking<double, unsigned long long>(p, st) : launch_ranking<float, unsigned>(p, st);
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------ Sim(3) alignment
namespace {

// The partials of the three passes and the solved transform.  Its size does not depend on n.
ovg::Sim3Params sim3_layout(Arena& ar) {
  ovg::Sim3Params p{};
  p.part0 = ar.get<double>(ovg::SIM3_BLOCKS * ovg::SIM3_P0);
  p.part1 = ar.get<double>(ovg::SIM3_BLOCKS * ovg::SIM3_P1);
  p.part2 = ar.get<double>(ovg::SIM3_BLOCKS);
  p.solved = ar.get<double>(12);
  return p;
}

}  // namespace

extern "C" {

long long ovg_sim3_workspace_bytes(long long n) {
  return n >= 0 ? layout_bytes(sim3_layout) : -1;
}

int ovg_sim3_estimate(const float* src, const float* dst, const unsigned char* keep, long long n, void* workspace,
                      long long workspace_bytes, double* out_sim3, double* out_stats, void* stream) {
  OVG_REQUIRE(n >= 0, "n must be >= 0");
  OVG_REQUIRE((src && dst) || n == 0, "null src / dst");
  OVG_REQUIRE(out_sim3 && out_stats, "null out_sim3 / out_stats");
  ovg::Sim3Params p;
  int rc = carve(__func__, "ovg_sim3_workspace_bytes(n)", workspace, workspace_bytes, &p, sim3_layout);
  if (rc) return rc;
  p.src = src; p.dst = dst; p.keep = keep; p.n = n; p.sim3 = out_sim3; p.stats = out_stats;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ovg::sim3_means_kernel<<<ovg::SIM3_BLOCKS, ovg::SIM3_THREADS, 0, st>>>(p);
  rc = post_launch("ovg_sim3_estimate(means)");
  if (rc) return rc;
  ovg::sim3_moments_kernel<<<ovg::SIM3_BLOCKS, ovg::SIM3_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_sim3_estimate(moments)"))) return rc;
  ovg::sim3_solve_kernel<<<1, 32, 0, st>>>(p);
  if ((rc = post_launch("ovg_sim3_estimate(solve)"))) return rc;
  ovg::sim3_residual_kernel<<<ovg::SIM3_BLOCKS, ovg::SIM3_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_sim3_estimate(residual)"))) return rc;
  ovg::sim3_finish_kernel<<<1, 32, 0, st>>>(p);
  return post_launch("ovg_sim3_estimate(finish)");
}

int ovg_sim3_apply(const double* sim3, int views, long long hw, const float* points_in, float* points_out,
                   const float* points2_in, float* points2_out, const float* depth_in, float* depth_out,
                   const float* ext_in, float* ext_out, void* stream) {
  OVG_REQUIRE(sim3 && views > 0 && hw > 0, "bad arguments");
  OVG_REQUIRE(!points_in == !points_out && !points2_in == !points2_out && !depth_in == !depth_out && !ext_in == !ext_out,
              "each input needs its output and each output its input");
  ovg::Sim3ApplyParams p{sim3, {points_in, points2_in}, {points_out, points2_out}, depth_in, depth_out, ext_in, ext_out,
                         static_cast<long long>(views) * hw, views};
  long long blocks = (p.n_pix + 255) / 256;
  if (blocks > num_sms() * 8LL) blocks = num_sms() * 8LL;          // grid-stride inside
  ovg::sim3_apply_kernel<<<static_cast<int>(blocks), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return post_launch("ovg_sim3_apply");
}

}  // extern "C"

// -------------------------------------------------------------------------------------------------------------- evaluation
namespace {

struct EvalPoseBufs {
  void* sim3;                        // ovg_sim3_workspace_bytes
  ovg::EvalPoseParams p;
};

EvalPoseBufs eval_pose_layout(Arena& ar, int m) {
  EvalPoseBufs w;
  w.sim3 = ar.take(layout_bytes(sim3_layout));
  ovg::EvalPoseParams& p = w.p;
  p = ovg::EvalPoseParams{};
  p.m = m;
  p.keep = ar.get<unsigned char>(m);
  p.centre_gt = ar.get<float>(3LL * m);
  p.centre_pred = ar.get<float>(3LL * m);
  p.count = ar.get<int>(1);
  p.vidx = ar.get<int>(m);
  p.pose_gt = ar.get<double>(15LL * m);
  p.pose_pred = ar.get<double>(15LL * m);
  p.pair_counts = ar.get<unsigned int>(static_cast<long long>(ovg::EVAL_PAIR_BLOCKS) * ovg::EVAL_PAIR_COUNTS);
  return w;
}

// The selection region, the two medians' results and weights, and the partials of the depth group
struct EvalDepthBufs {
  void* select;                      // OVG_PERCENTILE_WORKSPACE_BYTES
  ovg::EvalDepthParams p;
};

EvalDepthBufs eval_depth_layout(Arena& ar, int S, long long hw) {
  EvalDepthBufs w;
  ovg::EvalDepthParams& p = w.p;
  p = ovg::EvalDepthParams{};
  p.S = S; p.hw = hw;
  p.tiles = static_cast<int>(ovg::compact_tiles(hw));
  p.ld = (S * hw + 3) / 4 * 4;
  w.select = ar.take(OVG_PERCENTILE_WORKSPACE_BYTES);
  p.sel = ar.get<float>(6);
  p.weight = ar.get<float>(2);
  p.count = ar.get<unsigned long long>(1);
  p.cols = ar.get<float>(2 * p.ld);
  p.part = ar.get<double>(static_cast<long long>(S) * p.tiles * ovg::EVAL_DEPTH_P);
  p.view_tot = ar.get<double>(static_cast<long long>(S) * ovg::EVAL_DEPTH_P);
  return w;
}

struct EvalPointsBufs {
  void* select;                      // OVG_PERCENTILE_WORKSPACE_BYTES
  ovg::EvalPointsParams p;
};

EvalPointsBufs eval_points_layout(Arena& ar, int S, int H, int W) {
  EvalPointsBufs w;
  ovg::EvalPointsParams& p = w.p;
  p = ovg::EvalPointsParams{};
  p.S = S; p.H = H; p.W = W;
  const long long n = static_cast<long long>(S) * H * W;
  p.ld = (n + 3) / 4 * 4;
  w.select = ar.take(OVG_PERCENTILE_WORKSPACE_BYTES);
  p.sel = ar.get<float>(6);
  p.weight = ar.get<float>(2);
  p.count = ar.get<unsigned long long>(2);
  p.normals = ar.get<double>(6 * n);
  p.cols = ar.get<float>(2 * p.ld);
  p.part = ar.get<double>(2LL * ovg::EVAL_DIST_BLOCKS * 3);
  return w;
}

// The two medians of a group: numpy.percentile(cols[j, :count[j]], 50) for j = 0, 1, where every column holds +inf past its
// values (so the ranks, which stay below the count, never reach them).  sel[3 j .. 3 j + 1] and weight[j] get the result.
int eval_medians(const float* cols, long long ld, const unsigned long long* count, int count_stride, void* select, float* sel,
                 float* weight, const char* what, cudaStream_t st) {
  const PercentileRegion r = percentile_region(select);
  for (int j = 0; j < 2; ++j) {
    ovg::eval_select_init_kernel<<<1, 128, 0, st>>>(r.state, r.hist, count + j * count_stride, 50.f, weight + j);
    int rc = post_launch((std::string(what) + "(median init)").c_str());
    if (rc) return rc;
    if ((rc = radix_select_passes(cols + j * ld, ld, select, sel + 3 * j, nullptr, what, st))) return rc;
  }
  return OVG_OK;
}

}  // namespace

extern "C" {

long long ovg_eval_pose_workspace_bytes(int m) {
  return (m > 0 && m <= ovg::EVAL_MAX_VIEWS) ? layout_bytes(eval_pose_layout, m) : -1;
}

int ovg_eval_pose(const float* gt_ext, const float* gt_intr, const float* pred_ext, const int* views, int m, void* workspace,
                  long long workspace_bytes, double* sim3_out, double* stats_out, int* pairs_out, double* pair_errors_out,
                  double* rpe_out, double* scores_out, void* stream) {
  OVG_REQUIRE(m > 0 && m <= ovg::EVAL_MAX_VIEWS, "m must be in [1, 8192]");
  EvalPoseBufs w;
  int rc = carve(__func__, "ovg_eval_pose_workspace_bytes(m)", workspace, workspace_bytes, &w, eval_pose_layout, m);
  if (rc) return rc;
  OVG_REQUIRE(gt_ext && gt_intr && pred_ext && views && sim3_out && stats_out && pairs_out && pair_errors_out && rpe_out &&
                  scores_out, "null operand");
  ovg::EvalPoseParams& p = w.p;
  p.gt_ext = gt_ext; p.gt_intr = gt_intr; p.pred_ext = pred_ext; p.views = views;
  p.sim3 = sim3_out; p.stats = stats_out; p.pairs_out = pairs_out; p.pair_err = pair_errors_out; p.rpe = rpe_out;
  p.scores = scores_out;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ovg::eval_pose_prep_kernel<<<1, 1024, 0, st>>>(p);
  if ((rc = post_launch("ovg_eval_pose(prep)"))) return rc;
  // the ATE alignment (vo_eval.py:190-199): Umeyama of the predicted centres onto the ground-truth ones
  if ((rc = ovg_sim3_estimate(p.centre_pred, p.centre_gt, p.keep, m, w.sim3, layout_bytes(sim3_layout), sim3_out, stats_out,
                              stream)))
    return rc;
  ovg::eval_rpe_kernel<<<(m + ovg::EVAL_THREADS - 1) / ovg::EVAL_THREADS, ovg::EVAL_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_eval_pose(rpe)"))) return rc;
  ovg::eval_pair_kernel<<<ovg::EVAL_PAIR_BLOCKS, ovg::EVAL_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_eval_pose(pairs)"))) return rc;
  ovg::eval_pose_finish_kernel<<<1, ovg::EVAL_THREADS, 0, st>>>(p);
  return post_launch("ovg_eval_pose(finish)");
}

long long ovg_eval_depth_workspace_bytes(int S, long long hw) {
  return (S > 0 && hw > 0 && S * hw < (1LL << 31)) ? layout_bytes(eval_depth_layout, S, hw) : -1;
}

int ovg_eval_depth(const float* gt, const unsigned char* mask, const float* pred, const unsigned char* view_sel, int S,
                   long long hw, void* workspace, long long workspace_bytes, double* scores_out, double* view_abs_rel,
                   double* view_delta1, long long* view_pixels, void* stream) {
  OVG_REQUIRE(S > 0 && hw > 0 && S * hw < (1LL << 31), "need S > 0, hw > 0 and S hw < 2^31");
  EvalDepthBufs w;
  int rc = carve(__func__, "ovg_eval_depth_workspace_bytes(S, hw)", workspace, workspace_bytes, &w, eval_depth_layout, S, hw);
  if (rc) return rc;
  OVG_REQUIRE(gt && pred && view_sel && scores_out && view_abs_rel && view_delta1 && view_pixels, "null operand");
  ovg::EvalDepthParams& p = w.p;
  p.gt = gt; p.mask = mask; p.pred = pred; p.view_sel = view_sel;
  p.scores = scores_out; p.view_abs_rel = view_abs_rel; p.view_delta1 = view_delta1; p.view_pixels = view_pixels;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  OVG_CUDA(cudaMemsetAsync(p.count, 0, sizeof(unsigned long long), st));
  ovg::eval_depth_fill_kernel<<<select_blocks(p.ld), ovg::EVAL_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_eval_depth(fill)"))) return rc;
  if ((rc = eval_medians(p.cols, p.ld, p.count, 0, w.select, p.sel, p.weight,
                         "ovg_eval_depth", st)))
    return rc;
  ovg::eval_depth_partial_kernel<<<dim3(p.tiles, S), ovg::EVAL_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_eval_depth(partials)"))) return rc;
  ovg::eval_depth_finish_kernel<<<1, ovg::EVAL_THREADS, 0, st>>>(p);
  return post_launch("ovg_eval_depth(finish)");
}

int ovg_eval_points_keep(const float* gt_ext, const float* gt_intr, const float* gt_depth, const unsigned char* mask,
                         const float* pred_points, const unsigned char* view_sel, int S, long long hw, float* c2w_out,
                         unsigned char* keep_out, void* stream) {
  OVG_REQUIRE(S > 0 && hw > 0 && S * hw < (1LL << 31), "need S > 0, hw > 0 and S hw < 2^31");
  OVG_REQUIRE(gt_ext && gt_intr && gt_depth && pred_points && view_sel && c2w_out && keep_out, "null operand");
  const ovg::EvalKeepParams p{gt_ext, gt_intr, gt_depth, mask, pred_points, view_sel, S, hw, c2w_out, keep_out};
  ovg::eval_points_keep_kernel<<<select_blocks(S * hw), ovg::EVAL_THREADS, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p);
  return post_launch("ovg_eval_points_keep");
}

long long ovg_eval_points_workspace_bytes(int S, int H, int W) {
  return (S > 0 && H > 0 && W > 0 && static_cast<long long>(S) * H * W < (1LL << 30))
             ? layout_bytes(eval_points_layout, S, H, W) : -1;
}

int ovg_eval_points(const float* points, const unsigned char* keep, int S, int H, int W, const void* match_workspace,
                    long long match_workspace_bytes, void* workspace, long long workspace_bytes, double* acc_dist,
                    double* comp_dist, double* scores_out, void* stream) {
  OVG_REQUIRE(S > 0 && H > 0 && W > 0 && static_cast<long long>(S) * H * W < (1LL << 30), "need S H W < 2^30");
  const long long cap = static_cast<long long>(S) * H * W;
  ovg::MatchParams m;
  int rc = match_check(__func__, 2, cap, 1, match_workspace, match_workspace_bytes, &m);
  if (rc) return rc;
  EvalPointsBufs w;
  rc = carve(__func__, "ovg_eval_points_workspace_bytes(S, H, W)", workspace, workspace_bytes, &w, eval_points_layout, S, H, W);
  if (rc) return rc;
  OVG_REQUIRE(points && keep && acc_dist && comp_dist && scores_out, "null operand");
  ovg::EvalPointsParams& p = w.p;
  p.m = m; p.points = points; p.keep = keep;
  p.dist[0] = acc_dist; p.dist[1] = comp_dist; p.scores = scores_out;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  ovg::eval_normals_kernel<<<select_blocks(2 * cap), ovg::EVAL_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_eval_points(normals)"))) return rc;
  ovg::eval_points_dist_kernel<<<dim3(ovg::EVAL_DIST_BLOCKS, 2), ovg::EVAL_THREADS, 0, st>>>(p);
  if ((rc = post_launch("ovg_eval_points(distances)"))) return rc;
  if ((rc = eval_medians(p.cols, p.ld, p.count, 1, w.select, p.sel, p.weight,
                         "ovg_eval_points", st)))
    return rc;
  ovg::eval_points_finish_kernel<<<1, 32, 0, st>>>(p);
  return post_launch("ovg_eval_points(finish)");
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
  return plan ? layout_bytes(ovg::jpg::plan_layout, plan, static_cast<int>(plan->route.size())) : -1;
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
  OVG_REQUIRE(d_stream && d_out && (reinterpret_cast<uintptr_t>(d_stream) & 255) == 0, "stream must be 256-byte aligned");
  Workspace w;
  int rc = carve(__func__, "ovg_jpeg_plan_workspace_bytes()", workspace, workspace_bytes, &w, plan_layout, plan, n);
  if (rc) return rc;
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
    rc = post_launch("ovg_jpeg_decode(sync)");
    if (rc) return rc;
    int changed = 0;
    OVG_CUDA(cudaMemcpyAsync(&changed, w.changed, 4, cudaMemcpyDeviceToHost, st));
    OVG_CUDA(cudaStreamSynchronize(st));
    plan->rounds = static_cast<int>(r + 1);
    if (!changed) break;
  }
  const long long nsub_chunks = (plan->nsub + SCAN_CHUNK - 1) / SCAN_CHUNK;
  jpeg_count_scan_local_kernel<<<static_cast<unsigned>(nsub_chunks), SCAN_CHUNK, 0, st>>>(p);
  rc = post_launch("ovg_jpeg_decode(count scan)");
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
