// Internal declarations shared by the CUDA translation units of libalm_ocr.so.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <map>
#include <memory>
#include <tuple>
#include <unordered_map>
#include <string>
#include <vector>

#include "../../include/alm_ocr.h"

namespace alm {

typedef __nv_bfloat16 bf16;

struct AlmError {
  int code;
  std::string msg;
};

#define ALM_CHECK_CUDA(expr)                                                                      \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess)                                                                        \
      throw alm::AlmError{ALM_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e) + " (" + __FILE__ + \
                                            ":" + std::to_string(__LINE__) + ")"};                \
  } while (0)

#define ALM_REQUIRE(cond, code, message)                          \
  do {                                                            \
    if (!(cond)) throw alm::AlmError{(code), std::string(message) + " [" #cond "]"}; \
  } while (0)

// ---------------------------------------------------------------------------------------------
// bump allocator over one cudaMalloc'ed slab (activations); weights use their own slab
// ---------------------------------------------------------------------------------------------
struct Arena {
  char* base = nullptr;
  size_t cap = 0, off = 0, high = 0;
  void* alloc(size_t bytes) {
    size_t a = (off + 1023) & ~size_t(1023);
    if (a + bytes > cap)
      throw AlmError{ALM_ERR_OOM, "workspace arena exhausted: need " + std::to_string(a + bytes) + " of " +
                                      std::to_string(cap) + " bytes (raise alm_set_option workspace_mb)"};
    off = a + bytes;
    if (off > high) high = off;
    return base + a;
  }
  template <class T>
  T* get(size_t n) {
    return reinterpret_cast<T*>(alloc(n * sizeof(T)));
  }
  size_t mark() const { return off; }
  void release(size_t m) { off = m; }
};
// releases the arena back to the mark on every exit path (exceptions included)
struct ArenaScope {
  Arena& a;
  size_t mk;
  explicit ArenaScope(Arena& arena) : a(arena), mk(arena.off) {}
  ~ArenaScope() { a.release(mk); }
  ArenaScope(const ArenaScope&) = delete;
  ArenaScope& operator=(const ArenaScope&) = delete;
};

// K-major bf16 operand (hi/lo split pair), optionally batched over two batch dims.
struct Operand {
  const bf16* hi = nullptr;
  const bf16* lo = nullptr;  // may be null when the context runs single-pass bf16
  int rows = 0;              // per batch
  int K = 0;
  long ld = 0;               // row stride, elements (multiple of 8)
  int nb0 = 1, nb1 = 1;      // batch extents (1 + stride 0 == broadcast)
  long bs0 = 0, bs1 = 0;     // batch strides, elements (multiples of 8)
};

enum { ACT_NONE = 0, ACT_GELU = 1, ACT_RELU = 2 };
enum { BIAS_NONE = 0, BIAS_COL = 1, BIAS_ROW = 2 };

// out[orow, n] = act(alpha * acc + bias) + resid[rrow, n]
//   orow = out_map ? out_map[row] : row   (negative -> row is dropped)
//   rrow = resid_map ? resid_map[row] : orow
// Output is fp32 (out_f32) and/or a split bf16 pair (out_hi / out_lo) usable as the next GEMM's operand.
struct Epilogue {
  float* out_f32 = nullptr;
  bf16* out_hi = nullptr;
  bf16* out_lo = nullptr;
  long ldo = 0, obs0 = 0, obs1 = 0;  // fp32 and bf16 outputs share geometry
  int col_group = 0;                 // > 0: output column c goes to (c / col_group) * col_group_stride + c % col_group
  long col_group_stride = 0;         //      (head-major K/V caches written by ONE wide GEMM; col_group % 4 == 0)
  const float* bias = nullptr;
  int bias_mode = BIAS_NONE;
  long bias_bs0 = 0;  // per-batch(b0) bias stride
  const float* resid = nullptr;
  long ldr = 0, rbs0 = 0, rbs1 = 0;
  const int* out_map = nullptr;
  const int* resid_map = nullptr;
  int act = ACT_NONE;
  float alpha = 1.0f;
};

struct Ctx;

void gemm(Ctx* c, const Operand& A, const Operand& B, const Epilogue& E);

// ---------------------------------------------------------------------------------------------
// weights
// ---------------------------------------------------------------------------------------------
struct HostTensor {
  std::vector<float> f32;  // converted to fp32 on load
  bool placeholder = false;  // shape-only entry (data == NULL): zeros now, real values arrive by alm_broadcast_weights
  std::vector<int64_t> shape;
  size_t numel() const { return f32.size(); }
};

struct SplitW {  // [N, Kpad] row-major bf16 hi/lo, K padded to a multiple of 8 with zeros
  bf16* hi = nullptr;
  bf16* lo = nullptr;
  int N = 0, K = 0, ld = 0;
  Operand op() const {
    Operand o;
    o.hi = hi; o.lo = lo; o.rows = N; o.K = K; o.ld = ld;
    return o;
  }
};

struct OmniModel;
struct MgpModel;

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// Device slabs holding the converted weights.  Shared (ref-counted) between the contexts of one GPU that serve the
// same model (alm_share_weights): one copy of the ~0.9 GB of planes, any number of execution contexts.
struct WeightStore {
  int device = 0;
  std::vector<void*> slabs;
  std::vector<size_t> used;  // bytes bump-allocated in each slab (the weight broadcast sends exactly these)
  ~WeightStore() {
    int cur = 0;
    cudaGetDevice(&cur);
    cudaSetDevice(device);
    for (void* p : slabs) cudaFree(p);
    cudaSetDevice(cur);
  }
};

struct Ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  cudaStream_t stream2 = nullptr;  // second stream: the poly and rec decode loops overlap
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  cudaEvent_t ev_t[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};  // encode start/end, decode start, pt end, decode end
  bool timing_valid[2] = {false, false};
  int num_sms = 132;
  std::string err;
  Arena ws;
  size_t ws_bytes = size_t(24) << 30;
  int gemm_impl = 0;  // 0 = wgmma, 1 = SIMT debug kernel
  int nsplit = 3;     // 3 = bf16x3 split (fp32-class), 1 = single-pass bf16
  bool lo_unused = false;  // set inside mgp_forward in single-pass mode: no kernel of that path reads lo planes
  PFN_encodeTiled encode = nullptr;
  long launches = 0;  // kernels launched since last reset (gpu_launches in bench.py)
  // memoised TMA descriptors (see gemm.cu)
  struct TmapKey {
    const void* base; int K, rows; long ld; int nb0, nb1; long bs0, bs1; int box_rows; long plane;
    bool operator==(const TmapKey& o) const {
      return base == o.base && K == o.K && rows == o.rows && ld == o.ld && nb0 == o.nb0 && nb1 == o.nb1 &&
             bs0 == o.bs0 && bs1 == o.bs1 && box_rows == o.box_rows && plane == o.plane;
    }
  };
  struct TmapHash {
    size_t operator()(const TmapKey& k) const {
      size_t h = reinterpret_cast<size_t>(k.base);
      auto mix = [&h](size_t v) { h ^= v + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2); };
      mix(k.K); mix(k.rows); mix(static_cast<size_t>(k.ld)); mix(k.nb0); mix(k.nb1);
      mix(static_cast<size_t>(k.bs0)); mix(static_cast<size_t>(k.bs1)); mix(k.box_rows); mix(static_cast<size_t>(k.plane));
      return h;
    }
  };
  std::unordered_map<TmapKey, CUtensorMap, TmapHash> tmap_cache;
  std::map<std::tuple<const void*, int, long>, CUtensorMap> xattn_tmaps;  // K/V cache planes (xattn_tma.cu)
  // Co-scheduling of in-flight batches: every GEMM CTA needs a whole SM (227 KB of shared memory) for the
  // whole launch, so a full-width encoder GEMM shuts every other stream out.  enc_grid_cap / dec_grid_cap bound the
  // persistent GEMM grids of the encoder / the decode loops; decode_priority runs the decode loops on internal
  // high-priority streams so that their short kernels are dispatched ahead of the encoder's wide elementwise grids.
  int enc_grid_cap = 0, dec_grid_cap = 0;
  int gemm_grid_cap = 0;  // cap in force (set by omni_encode / omni_decode)
  int decode_priority = 0;
  // timing experiments only ("debug_skip" option): inside the decoder layers drop the launches of a kernel
  // class (bit 0 cross-attention, 1 linears, 2 LayerNorm, 3 self-attention).  Results are garbage by construction.
  int debug_skip = 0;
  bool skip_scope = false;
  bool skipped(int bit) const { return skip_scope && (debug_skip & bit); }
  cudaStream_t stream_hi = nullptr;  // internal high-priority stream for the decode loops
  cudaEvent_t ev_prio = nullptr;
  cudaEvent_t ev_order = nullptr;  // alm_stream_wait / alm_stream_release
  cudaEvent_t ev_block = nullptr;  // cudaEventBlockingSync event: host waits that sleep instead of spinning
  int small_grid_cap = 0;  // > 0: GEMM launches with <= 2*SMs tiles use at most this many CTAs
  int decode_streams = 2;  // 2 = poly and rec decode loops overlap on two streams, 1 = serial
  int use_graphs = 1;  // replay captured CUDA graphs for the per-token decode steps
  int joint_decode = 1;  // 0 = never run the polygon and recognition loops as one joint pass (the A/B reference)
  unsigned long long* trace_buf = nullptr;  // optional in-kernel GEMM timeline (alm_set_option "trace_gemm")
  int* trace_idx = nullptr;
  int trace_cap = 0;
  int sattn_wide = 1;  // CTA-per-(sequence, head) self-attention step when there are few sequences
  int xattn_wg = 1;  // 2 = 8-warp variant of the 64-query fused cross-attention (two key groups per block)
  int xattn_ctas_per_sm = 2;  // persistent grid of the fused cross-attention kernel
  int xattn_impl = 0;  // 0 = fused flash-style cross-attention (xattn.cu), 1 = score GEMM + softmax + P.V GEMM,
                       // 2 = fused, TMA + mbarrier pipeline (xattn_tma.cu)
  int fuse_ln_gemv = 1;  // point loop: 1 = the pre-LayerNorms run inside the following GEMV (13 fewer dependent launches per token)
  int kv_decoders = 3;  // number of decoders (pt, poly, rec order) whose cross-attention K/V caches alm_omni_encode fills
  int rec_topk = 0;     // alm_omni_set_rec_candidates: 0 = greedy outputs only, 1..8 = also the k best classes per rec step
  int rec_beams = 0;    // alm_omni_set_rec_beams: 0 = greedy recognition, 1..8 = beam width of the recognition loop
  float beam_alpha = 1.f;  // length penalty of the final beam ranking (score / len^alpha)
  bool rec_locations = false;  // alm_omni_set_rec_locations: also reduce every rec step's last-layer cross-attention
  // alm_omni_set_rec_charset: rec_cs_sets = 0 (off), else the sets rec_cs_allowed [n_sets][rec_cs_chars] and, when not
  // empty, the row sets rec_cs_rows [B][cap] of the next alm_omni_decode_at
  int rec_cs_sets = 0, rec_cs_chars = 0;
  std::vector<uint8_t> rec_cs_allowed;
  std::vector<int32_t> rec_cs_rows;
  int attn_impl = 0;   // ViT attention: 0 = fused flash-style mma.sync kernel (attn_tc.cu), 1 = GEMM + softmax + GEMM
  int wattn_impl = 3;  // 3 = persistent TMA-fed mma.sync kernel over head pairs (wattn_ms.cu; odd head counts fall back to 0), 0 = one CTA per (window, head), 1 = fp32 SIMT debug kernel
  // optional per-GEMM event timing (alm_set_option "profile_gemm" 1; read with alm_profile_read)
  int profile_gemm = 0;
  struct GemmRec { cudaEvent_t a, b; double flops; };
  std::vector<GemmRec> gemm_recs;
  OmniModel* omni = nullptr;
  MgpModel* mgp = nullptr;
  std::shared_ptr<WeightStore> wstore;
  // multi-GPU (comm.cu): an NCCL communicator (created by alm_comm_init or attached), used for ONE weight broadcast
  // at start-up and ONE all-gather of decoded sequences per batch
  void* comm = nullptr;
  bool own_comm = false;
  int comm_rank = 0, comm_world = 1;
  void* gather_buf = nullptr;
  size_t gather_cap = 0;
  // weight slab bump allocator
  char* wbase = nullptr;
  size_t wcap = 0, woff = 0;
  void* walloc(size_t bytes);
  void ensure_ws();
};

// weight helpers (weights.cu)
const HostTensor& need(const std::map<std::string, HostTensor>& m, const std::string& k);
float* upload_f32(Ctx* c, const float* h, size_t n);
SplitW upload_split(Ctx* c, const float* w, int N, int K, int Kpad);  // w is [N,K] row-major fp32; Kpad<=0 -> round up to 8
int* upload_i32(Ctx* c, const std::vector<int>& v);

// ---------------------------------------------------------------------------------------------
// elementwise / gather / attention kernels (kernels.cu)
// ---------------------------------------------------------------------------------------------
// Gather `nsrc` source rows of width Cs (fp32, row stride lds) into one row of width C = nsrc*Cs, optional
// LayerNorm over C, write fp32 and/or split bf16.  map[r*nsrc + s] = source row or -1 (zeros).
// zero_missing: a row whose (single) source is -1 is written as zeros *without* LN/affine ("pad after norm").
// rows_half > 0: rows from rows_half on take gamma2 / beta2 / add2 instead (the second decoder of a joint decoder pass).
void gather_ln(Ctx* c, const float* src, long lds, const int* map, int nsrc, int Cs, long rows, const float* gamma,
               const float* beta, float eps, bool zero_missing, const float* add, long ld_add, float* out_f32,
               long ldo_f32, bf16* out_hi, bf16* out_lo, long ldo_bf, bf16* out2_hi, bf16* out2_lo,
               float* out2_f32 = nullptr, long rows_half = 0, const float* gamma2 = nullptr,
               const float* beta2 = nullptr, const float* add2 = nullptr);

void gemv_rows(Ctx* c, const float* x, const float* x2, int n_split, long ldx, const float* W, const float* bias,
               const float* resid, long ldr, float* out, long ldo, int M, int N, int K, int act,
               const float* ln_g = nullptr, const float* ln_b = nullptr, float ln_eps = 0.f, const float* pos = nullptr,
               int pos_split = 0);

// Hc / Wc: canvas of the images (0: H / W); slots: canvas slot of each image (NULL: image b is slot b)
void im2col_patch4(Ctx* c, const float* img, int B, int H, int W, int Hp, int Wp, bf16* hi, bf16* lo, int Hc = 0,
                   int Wc = 0, const int* slots = nullptr);

void window_attention(Ctx* c, const float* qkv, int C, int heads, int nWh, int nWw, int B, int shift, int Hp, int Wp,
                      const float* bias_dense, bf16* out_hi, bf16* out_lo, float* out_f32);

// same, from the split-bf16 qkv planes the GEMM epilogue writes (q rows pre-scaled by WATTN_QSCALE at load time)
constexpr float WATTN_QSCALE = 0.17677669529663687f;  // 32 ** -0.5 (swin_transformer.py:130)
void window_attention_split(Ctx* c, const bf16* qkv_hi, const bf16* qkv_lo, int C, int heads, int nWh, int nWw, int B,
                            int shift, int Hp, int Wp, const float* bias_dense, bf16* out_hi, bf16* out_lo, float* out_f32);

// fused dense attention for <= 272 tokens x 64-wide heads on the tensor cores (attn_tc.cu)
void attention_tc(Ctx* c, const bf16* qkv_hi, const bf16* qkv_lo, long ld, int B, int T, int H, bf16* out_hi, bf16* out_lo,
                  float* out_f32, long ldo);

void window_attention_ms(Ctx* c, const bf16* qkv_hi, const bf16* qkv_lo, int C, int heads, int nWh, int nWw, int B, int shift,
                         int Hp, int Wp, const float* bias_dense, bf16* out_hi, bf16* out_lo, float* out_f32);

void split_rows(Ctx* c, const float* src, long lds, long rows, int C, bf16* hi, bf16* lo, long ldo);

void softmax_rows(Ctx* c, const float* s, long lds, long rows, int n, const uint8_t* kpm, int rows_per_mask,
                  long mask_ld, float* out_f32, bf16* out_hi, bf16* out_lo, long ldo);

// Kernel attributes (dynamic shared-memory opt-in, carve-out) are per DEVICE, and one process may hold a context per
// GPU, each driven by its own host thread: a once-flag must therefore be per device ordinal, not per process.
struct DeviceOnce {
  std::atomic<unsigned long long> done{0};  // bit d = attributes already set on device d (ordinals < 64)
  bool need() const {
    int d = 0;
    cudaGetDevice(&d);
    return ((done.load(std::memory_order_acquire) >> (d & 63)) & 1ull) == 0;
  }
  void mark() {
    int d = 0;
    cudaGetDevice(&d);
    done.fetch_or(1ull << (d & 63), std::memory_order_release);
  }
};

// Every kernel of the per-token decode loop asks for the same (maximum) shared-memory carve-out: consecutive kernels
// with different L1/shared splits force an SM reconfiguration (the SM must drain) between every pair of launches.
template <class F>
inline void pin_carveout(F* kernel) {
  cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
}
#define ALM_PIN_CARVEOUT(kernel)            \
  do {                                      \
    static alm::DeviceOnce pinned_;         \
    if (pinned_.need()) {                   \
      alm::pin_carveout(kernel);            \
      pinned_.mark();                       \
    }                                       \
  } while (0)

// comm.cu
void comm_unique_id(void* id128);
void comm_init(Ctx* c, const void* id128, int rank, int world);
void comm_attach(Ctx* c, void* nccl_comm, int rank, int world);
void comm_release(Ctx* c);
void comm_broadcast_weights(Ctx* c, int root);
void comm_gather(Ctx* c, const void* send, size_t bytes, void* recv_host);

void count_launch(Ctx* c, int n = 1);
void check_launch(const char* what);

}  // namespace alm
