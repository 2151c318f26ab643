// extern "C" surface of libalm_ocr.so (include/alm_ocr.h).  Nothing throws across this boundary.
#include <string.h>

#include <algorithm>
#include <cmath>
#include <type_traits>

#include "alm_internal.h"
#include "box_core.h"
#include "line_core.h"
#include "mgp.h"
#include "omni.h"
#include "pre.h"
#include "ptx.cuh"
#include "region_turn_core.h"

using namespace alm;

static_assert(ALM_BOX_CROP == box_core::GEOM_CROP && ALM_BOX_QUAD == box_core::GEOM_QUAD &&
                  ALM_BOX_CURVE == box_core::GEOM_CURVE, "box geometry kinds");

struct alm_ctx {
  Ctx c;
  void* dev_in = nullptr;  // staging for host-resident inputs
  size_t dev_in_bytes = 0;
  void* dev_mask = nullptr;
  size_t dev_mask_bytes = 0;
};

namespace {

template <class F>
int guarded(alm_ctx* h, F&& f) {
  if (!h) return ALM_ERR_INVALID;
  try {
    cudaSetDevice(h->c.device);
    f();
    h->c.err.clear();
    return ALM_OK;
  } catch (const AlmError& e) {
    h->c.err = e.msg;
    return e.code;
  } catch (const std::exception& e) {
    h->c.err = std::string("exception: ") + e.what();
    return ALM_ERR_INVALID;
  } catch (...) {
    h->c.err = "unknown exception";
    return ALM_ERR_INVALID;
  }
}

// for the entry points without a context: f returns the code
template <class F>
int guarded_free(F&& f) {
  try {
    return f();
  } catch (const AlmError& e) {
    return e.code;
  } catch (...) {
    return ALM_ERR_INVALID;
  }
}

bool is_device_ptr(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged;
}

// every non-null pointer is device memory aligned to `align` bytes
void require_device(std::initializer_list<const void*> ptrs, size_t align, const std::string& what) {
  for (const void* p : ptrs)
    ALM_REQUIRE(!p || (is_device_ptr(p) && reinterpret_cast<uintptr_t>(p) % align == 0), ALM_ERR_INVALID,
                what + (align > 1 ? ": device pointers aligned to " + std::to_string(align) + " bytes required"
                                  : std::string(": device pointers required")));
}

// milliseconds of `iters` calls of body() on the stream, after `warmup` untimed ones
template <class F>
float time_ms(Ctx* c, int warmup, int iters, F&& body) {
  for (int i = 0; i < warmup; ++i) body();
  cudaEvent_t e0, e1;
  ALM_CHECK_CUDA(cudaEventCreate(&e0));
  ALM_CHECK_CUDA(cudaEventCreate(&e1));
  ALM_CHECK_CUDA(cudaEventRecord(e0, c->stream));
  for (int i = 0; i < iters; ++i) body();
  ALM_CHECK_CUDA(cudaEventRecord(e1, c->stream));
  ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  float ms = 0;
  ALM_CHECK_CUDA(cudaEventElapsedTime(&ms, e0, e1));
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return ms;
}

// returns a device pointer for `p` (host buffers are copied into the context's staging slab on the stream)
const void* stage_input(alm_ctx* h, const void* p, size_t bytes, void** slab, size_t* slab_bytes) {
  if (p == nullptr) return nullptr;
  if (is_device_ptr(p)) return p;
  if (*slab_bytes < bytes) {
    if (*slab) cudaFree(*slab);
    *slab = nullptr;
    *slab_bytes = 0;
    if (cudaMalloc(slab, bytes) != cudaSuccess) throw AlmError{ALM_ERR_OOM, "cudaMalloc of the input staging buffer failed"};
    *slab_bytes = bytes;
  }
  ALM_CHECK_CUDA(cudaMemcpyAsync(*slab, p, bytes, cudaMemcpyHostToDevice, h->c.stream));
  return *slab;
}

// device copies of the caller's uint8 HWC images (host pointers are staged into the workspace on the stream)
std::vector<PreImage> stage_images(alm_ctx* h, const uint8_t* const* rgb, const int* heights, const int* widths, int n) {
  Ctx* c = &h->c;
  c->ensure_ws();
  std::vector<PreImage> imgs(static_cast<size_t>(n));
  for (int i = 0; i < n; ++i) {
    ALM_REQUIRE(rgb[i] && heights[i] > 0 && widths[i] > 0, ALM_ERR_INVALID, "image pointer / size");
    const size_t bytes = static_cast<size_t>(heights[i]) * widths[i] * 3;
    const uint8_t* d = rgb[i];
    if (!is_device_ptr(d)) {
      uint8_t* slot = c->ws.get<uint8_t>(bytes);
      ALM_CHECK_CUDA(cudaMemcpyAsync(slot, rgb[i], bytes, cudaMemcpyHostToDevice, c->stream));
      d = slot;
    }
    imgs[static_cast<size_t>(i)] = PreImage{d, heights[i], widths[i], 0, 0};
  }
  return imgs;
}

// body(pages) on the caller's pages staged by stage_images, once every output is known to be device memory; the pages
// live in the workspace until body returns
template <class F>
void with_pages(alm_ctx* h, const uint8_t* const* rgb, const int* heights, const int* widths, int n,
                std::initializer_list<const void*> outs, const char* what, F&& body) {
  require_device(outs, 1, std::string(what) + " outputs");
  Ctx* c = &h->c;
  c->ensure_ws();
  ArenaScope arena_scope(c->ws);
  std::vector<PreImage> pages = stage_images(h, rgb, heights, widths, n);
  body(pages);
}

void d2h(Ctx* c, void* dst, const void* src, size_t bytes) {
  ALM_CHECK_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->stream));
}

float bf16_bits_to_f32(uint16_t v) {
  uint32_t u = static_cast<uint32_t>(v) << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}
float f16_bits_to_f32(uint16_t v) {
  const uint32_t s = (v >> 15) & 1, e = (v >> 10) & 31, m = v & 1023;
  uint32_t u;
  if (e == 0) {
    if (m == 0) u = s << 31;
    else {
      int ee = -1;
      uint32_t mm = m;
      do { ++ee; mm <<= 1; } while ((mm & 1024) == 0);
      u = (s << 31) | ((127 - 15 - ee) << 23) | ((mm & 1023) << 13);
    }
  } else if (e == 31) u = (s << 31) | 0x7f800000u | (m << 13);
  else u = (s << 31) | ((e - 15 + 127) << 23) | (m << 13);
  float f;
  memcpy(&f, &u, 4);
  return f;
}

// Layouts of the decoder op entry points: fp32 x [nimg][M][512] (8 heads x 64) into the model's split-bf16 caches.
// K_c / V_c: [img][96 slices][M][64], head h in slice h of the base pointer's decoder layer.
__global__ void op_head_major_kernel(const float* __restrict__ x, int M, long n, bf16* __restrict__ hi,
                                     bf16* __restrict__ lo) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int col = static_cast<int>(i & 511), h = col >> 6, d = col & 63;
  const long row = i >> 9, img = row / M, key = row % M;
  const long o = ((img * 96 + h) * M + key) * 64 + d;
  split_bf16(x[i], hi[o], lo[o]);
}
// V^T: [img][6144][Mpad], feature f of the base pointer's decoder layer in row f; columns M..Mpad-1 are not written
__global__ void op_feature_major_kernel(const float* __restrict__ x, int M, int Mpad, long n, bf16* __restrict__ hi,
                                        bf16* __restrict__ lo) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int f = static_cast<int>(i & 511);
  const long row = i >> 9, img = row / M, key = row % M;
  const long o = (img * 6144 + f) * Mpad + key;
  split_bf16(x[i], hi[o], lo[o]);
}
__global__ void op_join_kernel(const bf16* __restrict__ hi, const bf16* __restrict__ lo, long n, float* __restrict__ out) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) out[i] = __bfloat162float(hi[i]) + __bfloat162float(lo[i]);
}
unsigned blocks256(long n) { return static_cast<unsigned>((n + 255) / 256); }

// The model's decoder caches for nimg_total images in the workspace: K (and V when v is given), with layer dl of images
// img0..img0+nimg-1 scattered head-major from x [nimg_total][M][512].  Every element a call must not read holds NaN
// (0xffff): other layers, other images, and the keys at or past key_len[i] of image i (when key_len is given).
struct DecoderCache {
  bf16 *kh = nullptr, *kl = nullptr, *vh = nullptr, *vl = nullptr;
  long off = 0;  // elements from a plane's base to (img0, dl)
};
DecoderCache decoder_cache(Ctx* c, const float* k, const float* v, int nimg_total, int img0, int nimg, int M, int dl,
                           const int* key_len) {
  DecoderCache d;
  const size_t cache = static_cast<size_t>(nimg_total) * 96 * M * 64;
  d.kh = c->ws.get<bf16>(cache); d.kl = c->ws.get<bf16>(cache);
  if (v) { d.vh = c->ws.get<bf16>(cache); d.vl = c->ws.get<bf16>(cache); }
  for (bf16* p : {d.kh, d.kl, d.vh, d.vl})
    if (p) ALM_CHECK_CUDA(cudaMemsetAsync(p, 0xff, cache * 2, c->stream));
  d.off = (static_cast<long>(img0) * 96 + dl * 8) * M * 64;
  const long nkv = static_cast<long>(nimg) * M * 512, in_off = static_cast<long>(img0) * M * 512;
  op_head_major_kernel<<<blocks256(nkv), 256, 0, c->stream>>>(k + in_off, M, nkv, d.kh + d.off, d.kl + d.off);
  if (v) op_head_major_kernel<<<blocks256(nkv), 256, 0, c->stream>>>(v + in_off, M, nkv, d.vh + d.off, d.vl + d.off);
  check_launch("op_head_major");
  for (int i = 0; key_len && i < nimg; ++i) {
    const int n = key_len[img0 + i];
    if (n == M) continue;
    // rows n..M-1 of the 8 [M][64] head blocks of this image and layer
    const long base = d.off + static_cast<long>(i) * 96 * M * 64 + static_cast<long>(n) * 64;
    for (bf16* p : {d.kh, d.kl, d.vh, d.vl})
      if (p)
        ALM_CHECK_CUDA(cudaMemset2DAsync(p + base, static_cast<size_t>(M) * 128, 0xff, static_cast<size_t>(M - n) * 128, 8,
                                         c->stream));
  }
  return d;
}

}  // namespace

extern "C" {

const char* alm_version(void) { return "alm_ocr 0.1 (sm_90a, wgmma)"; }

int alm_init(int device, void* stream, alm_ctx** out) {
  if (!out) return ALM_ERR_INVALID;
  *out = nullptr;
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || device < 0 || device >= n) {
    cudaGetLastError();
    return ALM_ERR_CUDA;  // no CUDA device: the library has no CPU fallback
  }
  alm_ctx* h = new alm_ctx();
  h->c.device = device;
  int rc = guarded(h, [&] {
    ALM_CHECK_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    ALM_CHECK_CUDA(cudaGetDeviceProperties(&prop, device));
    ALM_REQUIRE(prop.major == 9 && prop.minor == 0, ALM_ERR_UNSUPPORTED,
                "libalm_ocr is built for sm_90a only; device is sm_" + std::to_string(prop.major) + std::to_string(prop.minor));
    h->c.num_sms = prop.multiProcessorCount;
    if (stream) h->c.stream = static_cast<cudaStream_t>(stream);
    else {
      ALM_CHECK_CUDA(cudaStreamCreateWithFlags(&h->c.stream, cudaStreamNonBlocking));
      h->c.own_stream = true;
    }
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    ALM_CHECK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    ALM_REQUIRE(fn != nullptr && q == cudaDriverEntryPointSuccess, ALM_ERR_CUDA, "cuTensorMapEncodeTiled not available");
    h->c.encode = reinterpret_cast<PFN_encodeTiled>(fn);
  });
  if (rc != ALM_OK) {
    delete h;
    return rc;
  }
  *out = h;
  return ALM_OK;
}

void alm_free(alm_ctx* h) {
  if (!h) return;
  cudaSetDevice(h->c.device);
  cudaStreamSynchronize(h->c.stream);
  delete h->c.omni;
  mgp_free(h->c.mgp);
  comm_release(&h->c);
  if (h->c.gather_buf) cudaFree(h->c.gather_buf);
  h->c.wstore.reset();  // frees the slabs when this was the last context using them
  if (h->c.ws.base) cudaFree(h->c.ws.base);
  if (h->dev_in) cudaFree(h->dev_in);
  if (h->dev_mask) cudaFree(h->dev_mask);
  if (h->c.stream2) cudaStreamDestroy(h->c.stream2);
  if (h->c.stream_hi) cudaStreamDestroy(h->c.stream_hi);
  if (h->c.ev_prio) cudaEventDestroy(h->c.ev_prio);
  if (h->c.ev_block) cudaEventDestroy(h->c.ev_block);
  if (h->c.ev_order) cudaEventDestroy(h->c.ev_order);
  if (h->c.ev_fork) { cudaEventDestroy(h->c.ev_fork); cudaEventDestroy(h->c.ev_join); }
  for (auto e : h->c.ev_t) if (e) cudaEventDestroy(e);
  if (h->c.own_stream) cudaStreamDestroy(h->c.stream);
  delete h;
}

const char* alm_last_error(const alm_ctx* h) { return h ? h->c.err.c_str() : "null context"; }

namespace {

// the integer options of alm_set_option
enum OptionKind { OPT_ANY, OPT_FLAG, OPT_SET };  // stored as given / stored as 0 or 1 / one of the values in `accepted`
struct IntOption {
  const char* name;
  int Ctx::*field;
  OptionKind kind;
  unsigned accepted;  // OPT_SET: bit v set when value v is accepted
  const char* rule;   // OPT_SET: the accepted values, for the error message
};
const IntOption kIntOptions[] = {
    {"nsplit", &Ctx::nsplit, OPT_SET, 0b1010, "1 or 3"},
    {"gemm_impl", &Ctx::gemm_impl, OPT_SET, 0b11, "0 or 1"},
    {"xattn_impl", &Ctx::xattn_impl, OPT_SET, 0b111, "0..2"},
    {"fuse_ln_gemv", &Ctx::fuse_ln_gemv, OPT_FLAG, 0, nullptr},
    {"kv_decoders", &Ctx::kv_decoders, OPT_SET, 0b1110, "1..3"},
    {"attn_impl", &Ctx::attn_impl, OPT_SET, 0b11, "0 or 1"},
    {"wattn_impl", &Ctx::wattn_impl, OPT_SET, 0b1011, "0, 1 or 3"},
    {"enc_grid_cap", &Ctx::enc_grid_cap, OPT_ANY, 0, nullptr},
    {"dec_grid_cap", &Ctx::dec_grid_cap, OPT_ANY, 0, nullptr},
    {"xattn_ctas_per_sm", &Ctx::xattn_ctas_per_sm, OPT_SET, 0b1110, "1..3"},
    {"xattn_wg", &Ctx::xattn_wg, OPT_SET, 0b110, "1 or 2"},
    {"sattn_wide", &Ctx::sattn_wide, OPT_FLAG, 0, nullptr},
    {"debug_skip", &Ctx::debug_skip, OPT_ANY, 0, nullptr},
    {"decode_priority", &Ctx::decode_priority, OPT_FLAG, 0, nullptr},
    {"small_grid_cap", &Ctx::small_grid_cap, OPT_ANY, 0, nullptr},
    {"decode_streams", &Ctx::decode_streams, OPT_SET, 0b110, "1 or 2"},
    {"use_graphs", &Ctx::use_graphs, OPT_FLAG, 0, nullptr},
    {"joint_decode", &Ctx::joint_decode, OPT_FLAG, 0, nullptr},
    {"profile_gemm", &Ctx::profile_gemm, OPT_FLAG, 0, nullptr},
};

}  // namespace

int alm_set_option(alm_ctx* h, const char* key, long value) {
  return guarded(h, [&] {
    const std::string k = key ? key : "";
    for (const IntOption& o : kIntOptions) {
      if (k != o.name) continue;
      ALM_REQUIRE(o.kind != OPT_SET || (value >= 0 && value < 32 && (o.accepted >> value & 1u)), ALM_ERR_INVALID,
                  k + " must be " + o.rule);
      h->c.*o.field = o.kind == OPT_FLAG ? (value ? 1 : 0) : static_cast<int>(value);
      return;
    }
    if (k == "trace_gemm") {
      if (h->c.trace_buf) { cudaFree(h->c.trace_buf); cudaFree(h->c.trace_idx); h->c.trace_buf = nullptr; h->c.trace_idx = nullptr; }
      h->c.trace_cap = static_cast<int>(value);
      if (value > 0) {
        ALM_CHECK_CUDA(cudaMalloc(&h->c.trace_buf, static_cast<size_t>(value) * 6 * sizeof(unsigned long long)));
        ALM_CHECK_CUDA(cudaMalloc(&h->c.trace_idx, sizeof(int)));
        ALM_CHECK_CUDA(cudaMemset(h->c.trace_idx, 0, sizeof(int)));
      }
    } else if (k == "workspace_mb") {
      ALM_REQUIRE(value >= 64 && h->c.ws.base == nullptr, ALM_ERR_STATE, "workspace_mb must be set before first use");
      h->c.ws_bytes = static_cast<size_t>(value) << 20;
    } else {
      throw AlmError{ALM_ERR_INVALID, "unknown option " + k};
    }
  });
}

long alm_launch_count(alm_ctx* h, int reset) {
  if (!h) return -1;
  const long n = h->c.launches;
  if (reset) h->c.launches = 0;
  return n;
}

int alm_profile_read(alm_ctx* h, double* gemm_ms, double* gemm_flops, long* gemm_launches) {
  return guarded(h, [&] {
    ALM_CHECK_CUDA(cudaStreamSynchronize(h->c.stream));
    double ms = 0, fl = 0;
    for (auto& r : h->c.gemm_recs) {
      float t = 0;
      ALM_CHECK_CUDA(cudaEventElapsedTime(&t, r.a, r.b));
      ms += t;
      fl += r.flops;
      cudaEventDestroy(r.a);
      cudaEventDestroy(r.b);
    }
    if (gemm_ms) *gemm_ms = ms;
    if (gemm_flops) *gemm_flops = fl;
    if (gemm_launches) *gemm_launches = static_cast<long>(h->c.gemm_recs.size());
    h->c.gemm_recs.clear();
  });
}

int alm_trace_read(alm_ctx* h, unsigned long long* out, int max_records, int* n_records) {
  return guarded(h, [&] {
    ALM_REQUIRE(h->c.trace_buf && out && n_records, ALM_ERR_STATE, "trace_gemm is not enabled");
    ALM_CHECK_CUDA(cudaStreamSynchronize(h->c.stream));
    int n = 0;
    ALM_CHECK_CUDA(cudaMemcpy(&n, h->c.trace_idx, sizeof(int), cudaMemcpyDeviceToHost));
    n = std::min(n, std::min(h->c.trace_cap, max_records));
    ALM_CHECK_CUDA(cudaMemcpy(out, h->c.trace_buf, static_cast<size_t>(n) * 6 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    ALM_CHECK_CUDA(cudaMemset(h->c.trace_idx, 0, sizeof(int)));
    *n_records = n;
  });
}

int alm_bench_graph_floor(alm_ctx* h, int nodes, int iters, float* us_per_node) {
  // replay cost of a captured chain of `nodes` trivial dependent kernels: the per-kernel floor of the decode loop
  return guarded(h, [&] {
    ALM_REQUIRE(nodes > 0 && iters > 0 && us_per_node, ALM_ERR_INVALID, "alm_bench_graph_floor arguments");
    Ctx* c = &h->c;
    c->ensure_ws();
    ArenaScope arena_scope(c->ws);
    int* p = c->ws.get<int>(4);
    ALM_CHECK_CUDA(cudaMemsetAsync(p, 0, 16, c->stream));
    cudaGraph_t g = nullptr;
    cudaGraphExec_t ge = nullptr;
    ALM_CHECK_CUDA(cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
    for (int i = 0; i < nodes; ++i) fill_i32(c, p, 1, i);
    ALM_CHECK_CUDA(cudaStreamEndCapture(c->stream, &g));
    ALM_CHECK_CUDA(cudaGraphInstantiate(&ge, g, 0));
    cudaGraphDestroy(g);
    const float ms = time_ms(c, 3, iters, [&] { ALM_CHECK_CUDA(cudaGraphLaunch(ge, c->stream)); });
    *us_per_node = ms * 1e3f / (static_cast<float>(iters) * nodes);
    cudaGraphExecDestroy(ge);
  });
}

int alm_bench_gemm_ex(alm_ctx* h, int M, int N, int K, int batch, int split_out, int act, int iters,
                      float* ms_per_launch, unsigned long long* detail_out /* reserved: NULL */) {
  return guarded(h, [&] {
    ALM_REQUIRE(M > 0 && N > 0 && K > 0 && K % 8 == 0 && batch > 0 && iters > 0 && ms_per_launch, ALM_ERR_INVALID,
                "alm_bench_gemm_ex arguments");
    ALM_REQUIRE(detail_out == nullptr, ALM_ERR_INVALID, "alm_bench_gemm_ex: detail_out is reserved and must be NULL");
    Ctx* c = &h->c;
    c->ensure_ws();
    ArenaScope arena_scope(c->ws);
    const size_t na = static_cast<size_t>(batch) * M * K, nb = static_cast<size_t>(batch) * N * K;
    const int ldo = (N + 7) & ~7;
    Operand a, b;
    bf16* ah = c->ws.get<bf16>(na); bf16* al = c->ws.get<bf16>(na);
    bf16* bh = c->ws.get<bf16>(nb); bf16* bl = c->ws.get<bf16>(nb);
    ALM_CHECK_CUDA(cudaMemsetAsync(ah, 0x3c, na * 2, c->stream)); ALM_CHECK_CUDA(cudaMemsetAsync(al, 0x30, na * 2, c->stream));
    ALM_CHECK_CUDA(cudaMemsetAsync(bh, 0x3c, nb * 2, c->stream)); ALM_CHECK_CUDA(cudaMemsetAsync(bl, 0x30, nb * 2, c->stream));
    a.hi = ah; a.lo = al; a.rows = M; a.K = K; a.ld = K; a.nb0 = batch; a.bs0 = static_cast<long>(M) * K;
    b.hi = bh; b.lo = bl; b.rows = N; b.K = K; b.ld = K; b.nb0 = batch; b.bs0 = static_cast<long>(N) * K;
    Epilogue e;
    const size_t no = static_cast<size_t>(batch) * M * ldo;
    if (split_out) { e.out_hi = c->ws.get<bf16>(no); e.out_lo = c->ws.get<bf16>(no); }
    else e.out_f32 = c->ws.get<float>(no);
    e.ldo = ldo; e.obs0 = static_cast<long>(M) * ldo; e.act = act;
    *ms_per_launch = time_ms(c, 3, iters, [&] { gemm(c, a, b, e); }) / iters;
  });
}

int alm_bench_gemm(alm_ctx* h, int M, int N, int K, int iters, float* ms_per_launch) {
  return guarded(h, [&] {
    ALM_REQUIRE(M > 0 && N > 0 && K > 0 && K % 8 == 0 && N % 8 == 0 && iters > 0 && ms_per_launch, ALM_ERR_INVALID,
                "alm_bench_gemm arguments");
    Ctx* c = &h->c;
    c->ensure_ws();
    ArenaScope arena_scope(c->ws);
    float* fa = c->ws.get<float>(static_cast<size_t>(M) * K);
    float* fb = c->ws.get<float>(static_cast<size_t>(N) * K);
    // any finite data does; reuse whatever the arena holds after clamping it through a split
    ALM_CHECK_CUDA(cudaMemsetAsync(fa, 0x3c, static_cast<size_t>(M) * K * 4, c->stream));
    ALM_CHECK_CUDA(cudaMemsetAsync(fb, 0x3c, static_cast<size_t>(N) * K * 4, c->stream));
    Operand a, b;
    bf16* ah = c->ws.get<bf16>(static_cast<size_t>(M) * K); bf16* al = c->ws.get<bf16>(static_cast<size_t>(M) * K);
    bf16* bh = c->ws.get<bf16>(static_cast<size_t>(N) * K); bf16* bl = c->ws.get<bf16>(static_cast<size_t>(N) * K);
    split_rows(c, fa, K, M, K, ah, al, K);
    split_rows(c, fb, K, N, K, bh, bl, K);
    a.hi = ah; a.lo = al; a.rows = M; a.K = K; a.ld = K;
    b.hi = bh; b.lo = bl; b.rows = N; b.K = K; b.ld = K;
    Epilogue e;
    e.out_f32 = c->ws.get<float>(static_cast<size_t>(M) * N);
    e.ldo = N;
    *ms_per_launch = time_ms(c, 3, iters, [&] { gemm(c, a, b, e); }) / iters;
  });
}

int alm_load_weights(alm_ctx* h, int model_kind, const alm_tensor_desc* tensors, int n) {
  return guarded(h, [&] {
    ALM_REQUIRE(tensors && n > 0, ALM_ERR_INVALID, "empty state dict");
    std::map<std::string, HostTensor> t;
    for (int i = 0; i < n; ++i) {
      const alm_tensor_desc& d = tensors[i];
      ALM_REQUIRE(d.name && d.ndim >= 0 && d.ndim <= 4, ALM_ERR_INVALID, "bad tensor descriptor");
      HostTensor ht;
      size_t numel = 1;
      for (int k = 0; k < d.ndim; ++k) {
        ht.shape.push_back(d.shape[k]);
        numel *= static_cast<size_t>(d.shape[k]);
      }
      ht.f32.resize(numel);
      if (d.data == nullptr) {  // shape-only placeholder (non-root ranks before alm_broadcast_weights)
        ht.placeholder = true;
        t.emplace(d.name, std::move(ht));
        continue;
      }
      switch (d.dtype) {
        case ALM_F32: memcpy(ht.f32.data(), d.data, numel * 4); break;
        case ALM_F16:
          for (size_t j = 0; j < numel; ++j) ht.f32[j] = f16_bits_to_f32(static_cast<const uint16_t*>(d.data)[j]);
          break;
        case ALM_BF16:
          for (size_t j = 0; j < numel; ++j) ht.f32[j] = bf16_bits_to_f32(static_cast<const uint16_t*>(d.data)[j]);
          break;
        case ALM_I64:
          for (size_t j = 0; j < numel; ++j) ht.f32[j] = static_cast<float>(static_cast<const int64_t*>(d.data)[j]);
          break;
        default: throw AlmError{ALM_ERR_INVALID, std::string("unknown dtype for ") + d.name};
      }
      t.emplace(d.name, std::move(ht));
    }
    if (model_kind == ALM_MODEL_OMNI_SPOT || model_kind == ALM_MODEL_OMNI_KIE) omni_load(&h->c, model_kind, t);
    else if (model_kind == ALM_MODEL_MGPSTR) mgp_load(&h->c, t);
    else throw AlmError{ALM_ERR_INVALID, "unknown model kind"};
    ALM_CHECK_CUDA(cudaDeviceSynchronize());
  });
}

int alm_synchronize(alm_ctx* h) {
  return guarded(h, [&] { ALM_CHECK_CUDA(cudaStreamSynchronize(h->c.stream)); });
}

// ------------------------------------------------------------------------------------------ sharing / streams / comm
int alm_share_weights(alm_ctx* h, alm_ctx* owner) {
  return guarded(h, [&] {
    ALM_REQUIRE(owner && owner != h, ALM_ERR_INVALID, "alm_share_weights: owner context");
    ALM_REQUIRE(owner->c.device == h->c.device, ALM_ERR_INVALID, "alm_share_weights: contexts are on different devices");
    ALM_REQUIRE(owner->c.wstore && (owner->c.omni || owner->c.mgp), ALM_ERR_STATE, "alm_share_weights: owner has no weights");
    delete h->c.omni;
    h->c.omni = nullptr;
    mgp_free(h->c.mgp);
    h->c.mgp = nullptr;
    h->c.wstore = owner->c.wstore;  // ref-counted: the slabs live until the last context using them is freed
    h->c.wbase = nullptr; h->c.wcap = 0; h->c.woff = 0;
    if (owner->c.omni) h->c.omni = omni_share(owner->c.omni);
    if (owner->c.mgp) h->c.mgp = mgp_share(owner->c.mgp);
  });
}

int alm_stream_wait(alm_ctx* h, void* producer_stream) {
  return guarded(h, [&] {
    Ctx* c = &h->c;
    if (!c->ev_order) ALM_CHECK_CUDA(cudaEventCreateWithFlags(&c->ev_order, cudaEventDisableTiming));
    ALM_CHECK_CUDA(cudaEventRecord(c->ev_order, static_cast<cudaStream_t>(producer_stream)));
    ALM_CHECK_CUDA(cudaStreamWaitEvent(c->stream, c->ev_order, 0));
  });
}

int alm_stream_release(alm_ctx* h, void* consumer_stream) {
  return guarded(h, [&] {
    Ctx* c = &h->c;
    if (!c->ev_order) ALM_CHECK_CUDA(cudaEventCreateWithFlags(&c->ev_order, cudaEventDisableTiming));
    ALM_CHECK_CUDA(cudaEventRecord(c->ev_order, c->stream));
    ALM_CHECK_CUDA(cudaStreamWaitEvent(static_cast<cudaStream_t>(consumer_stream), c->ev_order, 0));
  });
}

int alm_comm_unique_id(void* id128) {
  if (!id128) return ALM_ERR_INVALID;
  return guarded_free([&] {
    comm_unique_id(id128);
    return ALM_OK;
  });
}

int alm_comm_init(alm_ctx* h, const void* id128, int rank, int world) {
  return guarded(h, [&] { comm_init(&h->c, id128, rank, world); });
}

int alm_comm_attach(alm_ctx* h, void* nccl_comm, int rank, int world) {
  return guarded(h, [&] { comm_attach(&h->c, nccl_comm, rank, world); });
}

int alm_broadcast_weights(alm_ctx* h, int root) {
  return guarded(h, [&] { comm_broadcast_weights(&h->c, root); });
}

int alm_gather_sequences(alm_ctx* h, const void* send, size_t bytes_per_rank, void* recv_host) {
  return guarded(h, [&] { comm_gather(&h->c, send, bytes_per_rank, recv_host); });
}

// ------------------------------------------------------------------------------------------ pre-processing
int alm_pre_omni_plan(const int* heights, const int* widths, int n, int test_min_size, int test_max_size, int* sizes,
                      int* Hmax, int* Wmax) {
  if (!heights || !widths || n < 0 || test_min_size <= 0 || !sizes || !Hmax || !Wmax) return ALM_ERR_INVALID;
  int hm = 0, wm = 0;
  for (int i = 0; i < n; ++i) {
    if (heights[i] <= 0 || widths[i] <= 0) return ALM_ERR_INVALID;
    pre_omni_size(heights[i], widths[i], test_min_size, test_max_size, &sizes[2 * i], &sizes[2 * i + 1]);
    hm = std::max(hm, sizes[2 * i]);
    wm = std::max(wm, sizes[2 * i + 1]);
  }
  *Hmax = hm; *Wmax = wm;
  return ALM_OK;
}

int alm_pre_coeffs(int in_size, int out_size, int filter, int* ksize, int* bounds, int* coefs, size_t cap_ints) {
  return guarded_free([&] { return pre_coeffs(in_size, out_size, filter, ksize, bounds, coefs, cap_ints); });
}

int alm_pre_omni_pages(alm_ctx* h, const uint8_t* const* rgb, const int* heights, const int* widths, int n,
                       int test_min_size, int test_max_size, float* tensors, uint8_t* mask) {
  return guarded(h, [&] {
    ALM_REQUIRE(rgb && heights && widths && n > 0 && test_min_size > 0 && tensors && mask, ALM_ERR_INVALID,
                "alm_pre_omni_pages arguments");
    with_pages(h, rgb, heights, widths, n, {tensors, mask}, "alm_pre_omni_pages", [&](std::vector<PreImage>& imgs) {
      int Hc = 0, Wc = 0;
      for (auto& im : imgs) {
        pre_omni_size(im.h, im.w, test_min_size, test_max_size, &im.oh, &im.ow);
        Hc = std::max(Hc, im.oh);
        Wc = std::max(Wc, im.ow);
      }
      pre_resize_batch(&h->c, imgs, PRE_BILINEAR, true, tensors, Hc, Wc, mask);
    });
  });
}

int alm_pre_mgp_crops(alm_ctx* h, const uint8_t* const* rgb, const int* heights, const int* widths, int n, int imgH,
                      int imgW, float* out) {
  return guarded(h, [&] {
    ALM_REQUIRE(rgb && heights && widths && n > 0 && imgH > 0 && imgW > 0 && out, ALM_ERR_INVALID,
                "alm_pre_mgp_crops arguments");
    with_pages(h, rgb, heights, widths, n, {out}, "alm_pre_mgp_crops", [&](std::vector<PreImage>& imgs) {
      for (auto& im : imgs) { im.oh = imgH; im.ow = imgW; }
      pre_resize_batch(&h->c, imgs, PRE_BICUBIC, false, out, imgH, imgW, nullptr);
    });
  });
}

int alm_pre_quad_plan(const int* heights, const int* widths, int n_pages, const float* quads, const int* page_index, int R,
                      float* ordered, float* corners, int* sizes, double* minv) {
  if (R == 0) return ALM_OK;
  if (!heights || !widths || n_pages < 1 || !quads || !page_index || R < 0) return ALM_ERR_INVALID;
  return guarded_free([&] {
    const std::vector<QuadPlan> plans = pre_quad_plan(heights, widths, n_pages, quads, page_index, R);
    for (int r = 0; r < R; ++r) {
      const QuadPlan& p = plans[static_cast<size_t>(r)];
      if (ordered) std::copy(p.ordered, p.ordered + 8, ordered + 8L * r);
      if (corners) std::copy(p.corners, p.corners + 8, corners + 8L * r);
      if (sizes) { sizes[2L * r] = p.cw; sizes[2L * r + 1] = p.ch; }
      if (minv) std::copy(p.mi, p.mi + 9, minv + 9L * r);
    }
    return ALM_OK;
  });
}

int alm_pre_quad_crops(alm_ctx* h, const uint8_t* const* rgb, const int* heights, const int* widths, int n_pages,
                       const float* quads, const int* page_index, int R, int imgH, int imgW, float* out) {
  return guarded(h, [&] {
    ALM_REQUIRE(R >= 0 && imgH > 0 && imgW > 0, ALM_ERR_INVALID, "alm_pre_quad_crops arguments");
    if (R == 0) return;
    ALM_REQUIRE(rgb && heights && widths && n_pages > 0 && quads && page_index && out, ALM_ERR_INVALID,
                "alm_pre_quad_crops arguments");
    const std::vector<QuadPlan> plans = pre_quad_plan(heights, widths, n_pages, quads, page_index, R);  // before any copy
    with_pages(h, rgb, heights, widths, n_pages, {out}, "alm_pre_quad_crops",
               [&](std::vector<PreImage>& pages) { pre_quad_crops(&h->c, pages, plans, imgH, imgW, out); });
  });
}

int alm_pre_curve_plan(const int* heights, const int* widths, int n_pages, const float* polys, const int* page_index,
                       int R, double* ctrl, int* sizes) {
  if (R == 0) return ALM_OK;
  if (!heights || !widths || n_pages < 1 || !polys || !page_index || R < 0) return ALM_ERR_INVALID;
  return guarded_free([&] {
    const std::vector<CurvePlan> plans = pre_curve_plan(heights, widths, n_pages, polys, page_index, R);
    for (int r = 0; r < R; ++r) {
      const CurvePlan& p = plans[static_cast<size_t>(r)];
      if (ctrl) std::copy(&p.ctrl[0][0][0], &p.ctrl[0][0][0] + 16, ctrl + 16L * r);
      if (sizes) { sizes[2L * r] = p.cw; sizes[2L * r + 1] = p.ch; }
    }
    return ALM_OK;
  });
}

int alm_pre_curve_crops(alm_ctx* h, const uint8_t* const* rgb, const int* heights, const int* widths, int n_pages,
                        const float* polys, const int* page_index, int R, int imgH, int imgW, float* out) {
  return guarded(h, [&] {
    ALM_REQUIRE(R >= 0 && imgH > 0 && imgW > 0, ALM_ERR_INVALID, "alm_pre_curve_crops arguments");
    if (R == 0) return;
    ALM_REQUIRE(rgb && heights && widths && n_pages > 0 && polys && page_index && out, ALM_ERR_INVALID,
                "alm_pre_curve_crops arguments");
    const std::vector<CurvePlan> plans = pre_curve_plan(heights, widths, n_pages, polys, page_index, R);  // before any copy
    with_pages(h, rgb, heights, widths, n_pages, {out}, "alm_pre_curve_crops",
               [&](std::vector<PreImage>& pages) { pre_curve_crops(&h->c, pages, plans, imgH, imgW, out); });
  });
}

int alm_pre_line_windows(const int* sizes, int R, int* n, int* x0, int* wn) {
  if (R == 0) return ALM_OK;
  if (!sizes || R < 0) return ALM_ERR_INVALID;
  for (int r = 0; r < R; ++r)
    if (sizes[2L * r] < 1 || sizes[2L * r + 1] < 1) return ALM_ERR_INVALID;
  for (int r = 0; r < R; ++r) {
    const line_core::Windows w = line_core::line_windows(sizes[2L * r], sizes[2L * r + 1]);
    if (n) n[r] = w.n;
    if (wn) wn[r] = w.wn;
    if (x0) std::copy(w.x0, w.x0 + line_core::kMaxWindows, x0 + static_cast<long>(line_core::kMaxWindows) * r);
  }
  return ALM_OK;
}

int alm_pre_line_crops(alm_ctx* h, const uint8_t* const* rgb, const int* heights, const int* widths, int n_pages,
                       int kind, const float* regions, const int* page_index, int R, float* out) {
  return guarded(h, [&] {
    ALM_REQUIRE(R >= 0, ALM_ERR_INVALID, "alm_pre_line_crops arguments");
    ALM_REQUIRE(kind == ALM_BOX_QUAD || kind == ALM_BOX_CURVE, ALM_ERR_INVALID,
                "alm_pre_line_crops: kind must be 1 (quad) or 2 (curve)");
    if (R == 0) return;
    ALM_REQUIRE(rgb && heights && widths && n_pages > 0 && regions && page_index && out, ALM_ERR_INVALID,
                "alm_pre_line_crops arguments");
    auto crops = [&](const auto& plans) {  // plans before any copy
      with_pages(h, rgb, heights, widths, n_pages, {out}, "alm_pre_line_crops",
                 [&](std::vector<PreImage>& pages) { pre_line_crops(&h->c, pages, plans, out); });
    };
    if (kind == ALM_BOX_QUAD) crops(pre_quad_plan(heights, widths, n_pages, regions, page_index, R));
    else crops(pre_curve_plan(heights, widths, n_pages, regions, page_index, R));
  });
}

namespace {

// every turn of a reading is a quarter-turn count 0..3
void require_turns(const int32_t* turns, int n, const char* fn) {
  for (int i = 0; i < n; ++i)
    ALM_REQUIRE(turns[i] >= 0 && turns[i] <= 3, ALM_ERR_INVALID,
                std::string(fn) + ": reading " + std::to_string(i) + ": turn " + std::to_string(turns[i]) +
                    " outside 0..3");
}

}  // namespace

int alm_pre_turned_crops(alm_ctx* h, const uint8_t* const* rgb, const int* heights, const int* widths, int n_pages,
                         int kind, const float* regions, const int* page_index, int R, const int32_t* turns, int lines,
                         float* out) {
  return guarded(h, [&] {
    const char* fn = "alm_pre_turned_crops";
    ALM_REQUIRE(R >= 0 && (lines == 0 || lines == 1), ALM_ERR_INVALID, std::string(fn) + " arguments");
    ALM_REQUIRE(kind == ALM_BOX_QUAD || kind == ALM_BOX_CURVE, ALM_ERR_INVALID,
                std::string(fn) + ": kind must be 1 (quad) or 2 (curve)");
    if (R == 0) return;
    ALM_REQUIRE(rgb && heights && widths && n_pages > 0 && regions && page_index && turns && out, ALM_ERR_INVALID,
                std::string(fn) + " arguments");
    require_turns(turns, R, fn);
    auto crops = [&](const auto& plans) {  // plans before any copy
      with_pages(h, rgb, heights, widths, n_pages, {out}, fn, [&](std::vector<PreImage>& pages) {
        constexpr bool quad = std::is_same<std::decay_t<decltype(plans)>, std::vector<QuadPlan>>::value;
        if (lines) pre_line_crops(&h->c, pages, plans, out, turns);
        else if constexpr (quad) pre_quad_crops(&h->c, pages, plans, box_core::kImgH, box_core::kImgW, out, turns);
        else pre_curve_crops(&h->c, pages, plans, box_core::kImgH, box_core::kImgW, out, turns);
      });
    };
    if (kind == ALM_BOX_QUAD) crops(pre_quad_plan(heights, widths, n_pages, regions, page_index, R));
    else crops(pre_curve_plan(heights, widths, n_pages, regions, page_index, R));
  });
}

namespace {

// the tiles of every page in plan order (page-major, row-major); T / ov already checked.  turns: null for upright
// pages, else [n_pages] in 0..3 (checked): page p is tiled as np.rot90(page, turns[p])
std::vector<tile_core::Tile> page_tiles(const int* heights, const int* widths, int n_pages, int T, int ov, double band,
                                        const int32_t* turns = nullptr) {
  std::vector<tile_core::Tile> tiles;
  for (int p = 0; p < n_pages; ++p) {
    const int first = static_cast<int>(tiles.size());
    const int k = turns ? turns[p] : 0;
    const int H = k & 1 ? widths[p] : heights[p], W = k & 1 ? heights[p] : widths[p];
    const long n = static_cast<long>(tile_core::axis_count(H, T, ov)) * tile_core::axis_count(W, T, ov);
    ALM_REQUIRE(first + n <= (1L << 20), ALM_ERR_INVALID, "more than 2^20 tiles");
    for (int i = 0; i < n; ++i)
      tiles.push_back(turns ? tile_core::make_turned_tile(p, first, heights[p], widths[p], k, T, ov, i, band)
                            : tile_core::make_tile(p, first, heights[p], widths[p], T, ov, i, band));
  }
  return tiles;
}

bool pages_ok(const int* heights, const int* widths, int n_pages) {
  if (!heights || !widths || n_pages < 1) return false;
  for (int p = 0; p < n_pages; ++p)
    if (heights[p] < 1 || widths[p] < 1) return false;
  return true;
}

}  // namespace

int alm_pre_omni_tile_plan(int H, int W, int tile, int overlap, int* ny, int* nx, int* y0, int* x0, int cap) {
  if (H < 1 || W < 1 || !tile_core::valid_layout(tile, overlap) || !ny || !nx) return ALM_ERR_INVALID;
  *ny = tile_core::axis_count(H, tile, overlap);
  *nx = tile_core::axis_count(W, tile, overlap);
  if (!y0 && !x0) return ALM_OK;
  if (cap < std::max(*ny, *nx)) return ALM_ERR_INVALID;
  for (int i = 0; y0 && i < *ny; ++i) y0[i] = tile_core::axis_origin(H, tile, overlap, i);
  for (int i = 0; x0 && i < *nx; ++i) x0[i] = tile_core::axis_origin(W, tile, overlap, i);
  return ALM_OK;
}

namespace {

// alm_pre_omni_tiles (turned false) / alm_pre_omni_tiles_turned / alm_pre_omni_tiles_at: the plan's tiles idx[0..n)
int omni_tiles(alm_ctx* h, const char* fn, const uint8_t* const* rgb, const int* heights, const int* widths, int n_pages,
               bool turned, const int32_t* turns, int tile, int overlap, const int32_t* idx, int count,
               int test_min_size, int test_max_size, float* tensors, uint8_t* mask) {
  return guarded(h, [&] {
    ALM_REQUIRE(rgb && pages_ok(heights, widths, n_pages) && tile_core::valid_layout(tile, overlap) &&
                    test_min_size > 0 && tensors && mask && (turns || !turned),
                ALM_ERR_INVALID, std::string(fn) + " arguments");
    if (turns) require_turns(turns, n_pages, fn);
    const std::vector<tile_core::Tile> tiles = page_tiles(heights, widths, n_pages, tile, overlap, 0.0, turns);
    ALM_REQUIRE(idx && count >= 1, ALM_ERR_INVALID, std::string(fn) + ": tile range outside the plan");
    for (int k = 0; k < count; ++k)
      ALM_REQUIRE(idx[k] >= 0 && idx[k] < static_cast<long>(tiles.size()), ALM_ERR_INVALID,
                  std::string(fn) + ": tile range outside the plan");
    with_pages(h, rgb, heights, widths, n_pages, {tensors, mask}, fn, [&](std::vector<PreImage>& pages) {
      std::vector<PreImage> imgs;
      tile_gather(&h->c, pages, tiles, std::vector<int>(idx, idx + count), &imgs);
      int Hc = 0, Wc = 0;
      for (PreImage& im : imgs) {
        pre_omni_size(im.h, im.w, test_min_size, test_max_size, &im.oh, &im.ow);
        Hc = std::max(Hc, im.oh);
        Wc = std::max(Wc, im.ow);
      }
      pre_resize_batch(&h->c, imgs, PRE_BILINEAR, true, tensors, Hc, Wc, mask);
    });
  });
}

// plan indices first .. first + count - 1; empty when count < 1 or the range reaches past any plan (2^20 tiles)
std::vector<int32_t> tile_range(int first, int count) {
  std::vector<int32_t> idx;
  if (count >= 1 && static_cast<long>(first) + count <= (1L << 20))
    for (int i = 0; i < count; ++i) idx.push_back(first + i);
  return idx;
}

}  // namespace

int alm_pre_omni_tiles(alm_ctx* h, const uint8_t* const* rgb, const int* heights, const int* widths, int n_pages,
                       int tile, int overlap, int first, int count, int test_min_size, int test_max_size, float* tensors,
                       uint8_t* mask) {
  const std::vector<int32_t> idx = tile_range(first, count);
  return omni_tiles(h, "alm_pre_omni_tiles", rgb, heights, widths, n_pages, false, nullptr, tile, overlap, idx.data(),
                    static_cast<int>(idx.size()), test_min_size, test_max_size, tensors, mask);
}

int alm_pre_omni_tiles_at(alm_ctx* h, const uint8_t* const* rgb, const int* heights, const int* widths, int n_pages,
                          int tile, int overlap, const int32_t* index, int count, int test_min_size, int test_max_size,
                          float* tensors, uint8_t* mask) {
  return omni_tiles(h, "alm_pre_omni_tiles_at", rgb, heights, widths, n_pages, false, nullptr, tile, overlap, index,
                    count, test_min_size, test_max_size, tensors, mask);
}

int alm_pre_omni_tiles_turned(alm_ctx* h, const uint8_t* const* rgb, const int* heights, const int* widths,
                              int n_pages, const int32_t* turns, int tile, int overlap, int first, int count,
                              int test_min_size, int test_max_size, float* tensors, uint8_t* mask) {
  const std::vector<int32_t> idx = tile_range(first, count);
  return omni_tiles(h, "alm_pre_omni_tiles_turned", rgb, heights, widths, n_pages, true, turns, tile, overlap,
                    idx.data(), static_cast<int>(idx.size()), test_min_size, test_max_size, tensors, mask);
}

int alm_pre_omni_tiles_at_turned(alm_ctx* h, const uint8_t* const* rgb, const int* heights, const int* widths,
                                 int n_pages, const int32_t* turns, int tile, int overlap, const int32_t* index,
                                 int count, int test_min_size, int test_max_size, float* tensors, uint8_t* mask) {
  return omni_tiles(h, "alm_pre_omni_tiles_at_turned", rgb, heights, widths, n_pages, true, turns, tile, overlap, index,
                    count, test_min_size, test_max_size, tensors, mask);
}

namespace {

// The tiles of a tile merge's plan (alm_omni_merge_tiles, _turned, alm_omni_merge_kie_tiles), once the page sizes, the
// layout, margin / band / iou, the turns (null: upright pages), n_tiles and every tile's page and origin are checked
std::vector<tile_core::Tile> merge_plan(const char* fn, const int* heights, const int* widths, int n_pages,
                                        const int32_t* turns, int tile, int overlap, double margin, double band,
                                        double iou, int n_tiles, const int* tile_page, const int* tile_origin) {
  ALM_REQUIRE(pages_ok(heights, widths, n_pages) && tile_core::valid_layout(tile, overlap), ALM_ERR_INVALID,
              std::string(fn) + ": page sizes, or tile size / overlap (need tile >= 64, 0 <= 2 overlap <= tile)");
  ALM_REQUIRE(std::isfinite(margin) && margin >= 0.0 && std::isfinite(band) && band >= 0.0 && std::isfinite(iou) &&
                  iou > 0.0 && iou <= 1.0,
              ALM_ERR_INVALID, std::string(fn) + ": margin and band must be finite and >= 0, iou in (0, 1]");
  ALM_REQUIRE(tile_page && tile_origin, ALM_ERR_INVALID, std::string(fn) + ": null argument");
  if (turns) require_turns(turns, n_pages, fn);
  std::vector<tile_core::Tile> tiles = page_tiles(heights, widths, n_pages, tile, overlap, band, turns);
  ALM_REQUIRE(n_tiles == static_cast<int>(tiles.size()), ALM_ERR_INVALID,
              std::string(fn) + ": " + std::to_string(n_tiles) + " tiles, the plan has " + std::to_string(tiles.size()));
  for (int k = 0; k < n_tiles; ++k) {
    const tile_core::Tile& t = tiles[static_cast<size_t>(k)];
    ALM_REQUIRE(tile_page[k] >= 0 && tile_page[k] < n_pages, ALM_ERR_INVALID,
                std::string(fn) + ": tile " + std::to_string(k) + ": page index out of range");
    ALM_REQUIRE(tile_page[k] == t.page && tile_origin[2 * k] == t.y0 && tile_origin[2 * k + 1] == t.x0,
                ALM_ERR_INVALID, std::string(fn) + ": tile " + std::to_string(k) + " is not the plan's tile " +
                                     std::to_string(k) + " (pages in order, tiles row-major)");
  }
  return tiles;
}

// The total of n counts, once every count is checked >= 0 and every offset the sum of the earlier counts; the
// refusals name each count `what` and its index
long prefix_total(const char* fn, const char* what, const int32_t* count, const int32_t* offset, long n) {
  long total = 0;
  for (long r = 0; r < n; ++r) {
    ALM_REQUIRE(count[r] >= 0, ALM_ERR_INVALID,
                std::string(fn) + ": " + what + " " + std::to_string(r) + ": negative count");
    ALM_REQUIRE(offset[r] == total, ALM_ERR_INVALID,
                std::string(fn) + ": " + what + " " + std::to_string(r) + ": offset is not the sum of the earlier counts");
    total += count[r];
  }
  return total;
}

// alm_omni_merge_tiles (turned false) / alm_omni_merge_tiles_turned
int merge_tiles(alm_ctx* h, const char* fn, const int* heights, const int* widths, int n_pages, bool turned,
                const int32_t* turns, int tile, int overlap, int n_tiles, const int* tile_page, const int* tile_origin,
                const int32_t* n_inst, const int64_t* pt, const int64_t* poly, const int64_t* rec,
                const float* rec_prob, int max_inst, int rec_length, int num_bins, double margin, double band,
                double iou, int* page_count, int* page_offset, double* pts, double* polys, int64_t* rec_out,
                float* prob_out, int32_t* source, long cap) {
  return guarded(h, [&] {
    ALM_REQUIRE(max_inst >= 1 && rec_length >= 1 && num_bins >= 1, ALM_ERR_INVALID,
                std::string(fn) + ": max_inst, rec_length and num_bins must be >= 1");
    ALM_REQUIRE(n_inst && pt && poly && rec && rec_prob && page_count && page_offset && (turns || !turned),
                ALM_ERR_INVALID, std::string(fn) + ": null argument");
    const std::vector<tile_core::Tile> tiles = merge_plan(fn, heights, widths, n_pages, turns, tile, overlap, margin,
                                                          band, iou, n_tiles, tile_page, tile_origin);
    long total = 0;
    for (int k = 0; k < n_tiles; ++k) {
      ALM_REQUIRE(n_inst[k] >= 0 && n_inst[k] <= max_inst, ALM_ERR_INVALID,
                  std::string(fn) + ": tile " + std::to_string(k) + ": n_inst outside [0, max_inst]");
      total += n_inst[k];
    }
    ALM_REQUIRE(cap >= total, ALM_ERR_INVALID, std::string(fn) + ": output capacity below the sum of n_inst");
    ALM_REQUIRE(total == 0 || (pts && polys && rec_out && prob_out && source), ALM_ERR_INVALID,
                std::string(fn) + ": null output buffer");
    tile_merge(&h->c, tiles, n_pages, max_inst, rec_length, num_bins, margin, iou, n_inst, pt, poly, rec, rec_prob,
               MergeRows{page_count, page_offset, pts, polys, rec_out, prob_out, source});
  });
}

}  // namespace

int alm_omni_merge_tiles(alm_ctx* h, const int* heights, const int* widths, int n_pages, int tile, int overlap,
                         int n_tiles, const int* tile_page, const int* tile_origin, const int32_t* n_inst,
                         const int64_t* pt, const int64_t* poly, const int64_t* rec, const float* rec_prob, int max_inst,
                         int rec_length, int num_bins, double margin, double band, double iou, int* page_count,
                         int* page_offset, double* pts, double* polys, int64_t* rec_out, float* prob_out,
                         int32_t* source, long cap) {
  return merge_tiles(h, "alm_omni_merge_tiles", heights, widths, n_pages, false, nullptr, tile, overlap, n_tiles,
                     tile_page, tile_origin, n_inst, pt, poly, rec, rec_prob, max_inst, rec_length, num_bins, margin,
                     band, iou, page_count, page_offset, pts, polys, rec_out, prob_out, source, cap);
}

int alm_omni_merge_tiles_turned(alm_ctx* h, const int* heights, const int* widths, int n_pages, const int32_t* turns,
                                int tile, int overlap, int n_tiles, const int* tile_page, const int* tile_origin,
                                const int32_t* n_inst, const int64_t* pt, const int64_t* poly, const int64_t* rec,
                                const float* rec_prob, int max_inst, int rec_length, int num_bins, double margin,
                                double band, double iou, int* page_count, int* page_offset, double* pts,
                                double* polys, int64_t* rec_out, float* prob_out, int32_t* source, long cap) {
  return merge_tiles(h, "alm_omni_merge_tiles_turned", heights, widths, n_pages, true, turns, tile, overlap, n_tiles,
                     tile_page, tile_origin, n_inst, pt, poly, rec, rec_prob, max_inst, rec_length, num_bins, margin,
                     band, iou, page_count, page_offset, pts, polys, rec_out, prob_out, source, cap);
}

int alm_omni_orient_select(alm_ctx* h, int n_pages, const int32_t* n_inst, const int64_t* rec, const float* rec_prob,
                           int max_inst, int rec_length, int recog_pad_index, int rec_eos_index, int32_t* turns_out,
                           double* scores) {
  return guarded(h, [&] {
    const char* fn = "alm_omni_orient_select";
    ALM_REQUIRE(n_pages >= 1 && max_inst >= 1 && rec_length >= 1, ALM_ERR_INVALID,
                std::string(fn) + ": n_pages, max_inst and rec_length must be >= 1");
    ALM_REQUIRE(n_inst && rec && rec_prob && turns_out && scores, ALM_ERR_INVALID, std::string(fn) + ": null argument");
    for (long r = 0; r < 4L * n_pages; ++r)
      ALM_REQUIRE(n_inst[r] >= 0 && n_inst[r] <= max_inst, ALM_ERR_INVALID,
                  std::string(fn) + ": reading " + std::to_string(r) + ": n_inst outside [0, max_inst]");
    orient_select(&h->c, n_pages, max_inst, rec_length, recog_pad_index, rec_eos_index, n_inst, rec, rec_prob,
                  turns_out, scores);
  });
}

namespace {

// alm_omni_merge_turns (nr = 4) and alm_omni_merge_readings: one set of checks, then reading_merge
int merge_readings(alm_ctx* h, const char* fn, int n_pages, int nr, const int32_t* count, const int32_t* offset,
                   const double* pts, const double* polys, const int64_t* rec, const float* rec_prob, int rec_length,
                   int recog_pad_index, int rec_eos_index, double iou, int32_t* page_count, int32_t* page_offset,
                   double* pts_out, double* polys_out, int64_t* rec_out, float* prob_out, int32_t* source, long cap) {
  return guarded(h, [&] {
    ALM_REQUIRE(n_pages >= 1 && rec_length >= 1, ALM_ERR_INVALID,
                std::string(fn) + ": n_pages and rec_length must be >= 1");
    ALM_REQUIRE(nr >= 1 && nr <= 64, ALM_ERR_INVALID, std::string(fn) + ": n_readings must be in 1..64");
    ALM_REQUIRE(count && offset && pts && polys && rec && rec_prob && page_count && page_offset && pts_out &&
                    polys_out && rec_out && prob_out && source,
                ALM_ERR_INVALID, std::string(fn) + ": null argument");
    ALM_REQUIRE(std::isfinite(iou) && iou > 0.0 && iou <= 1.0, ALM_ERR_INVALID,
                std::string(fn) + ": iou must be in (0, 1]");
    ALM_REQUIRE(static_cast<long>(nr) * n_pages <= INT_MAX / 2, ALM_ERR_INVALID, std::string(fn) + ": too many readings");
    const long total = prefix_total(fn, "reading", count, offset, static_cast<long>(nr) * n_pages);
    ALM_REQUIRE(total <= INT_MAX / 32, ALM_ERR_INVALID, std::string(fn) + ": too many rows");
    ALM_REQUIRE(cap >= total, ALM_ERR_INVALID, std::string(fn) + ": output capacity below the sum of the counts");
    reading_merge(&h->c, n_pages, nr, count, offset, rec_length, recog_pad_index, rec_eos_index, iou, pts, polys, rec,
                  rec_prob, MergeRows{page_count, page_offset, pts_out, polys_out, rec_out, prob_out, source});
  });
}

}  // namespace

int alm_omni_merge_turns(alm_ctx* h, int n_pages, const int32_t* count, const int32_t* offset, const double* pts,
                         const double* polys, const int64_t* rec, const float* rec_prob, int rec_length,
                         int recog_pad_index, int rec_eos_index, double iou, int32_t* page_count, int32_t* page_offset,
                         double* pts_out, double* polys_out, int64_t* rec_out, float* prob_out, int32_t* source,
                         long cap) {
  return merge_readings(h, "alm_omni_merge_turns", n_pages, 4, count, offset, pts, polys, rec, rec_prob, rec_length,
                        recog_pad_index, rec_eos_index, iou, page_count, page_offset, pts_out, polys_out, rec_out,
                        prob_out, source, cap);
}

int alm_omni_merge_readings(alm_ctx* h, int n_pages, int n_readings, const int32_t* count, const int32_t* offset,
                            const double* pts, const double* polys, const int64_t* rec, const float* rec_prob,
                            int rec_length, int recog_pad_index, int rec_eos_index, double iou, int32_t* page_count,
                            int32_t* page_offset, double* pts_out, double* polys_out, int64_t* rec_out,
                            float* prob_out, int32_t* source, long cap) {
  return merge_readings(h, "alm_omni_merge_readings", n_pages, n_readings, count, offset, pts, polys, rec, rec_prob,
                        rec_length, recog_pad_index, rec_eos_index, iou, page_count, page_offset, pts_out, polys_out,
                        rec_out, prob_out, source, cap);
}

int alm_omni_merge_whole_page(alm_ctx* h, const int* heights, const int* widths, int n_pages, const int32_t* turns,
                              int tile, int overlap, double margin, int num_bins, const int32_t* count,
                              const int32_t* offset, const double* pts, const double* polys, const int64_t* rec,
                              const float* rec_prob, const int32_t* source_in, const int32_t* n_inst, const int64_t* pt,
                              const int64_t* poly, const int64_t* whole_rec, const float* whole_prob, int cap_in,
                              int rec_length, int32_t* page_count, int32_t* page_offset, double* pts_out,
                              double* polys_out, int64_t* rec_out, float* prob_out, int32_t* source, long cap) {
  return guarded(h, [&] {
    const char* fn = "alm_omni_merge_whole_page";
    ALM_REQUIRE(pages_ok(heights, widths, n_pages) && tile_core::valid_layout(tile, overlap), ALM_ERR_INVALID,
                std::string(fn) + ": page sizes, or tile size / overlap (need tile >= 64, 0 <= 2 overlap <= tile)");
    ALM_REQUIRE(std::isfinite(margin) && margin >= 0.0, ALM_ERR_INVALID,
                std::string(fn) + ": margin must be finite and >= 0");
    ALM_REQUIRE(num_bins >= 1 && rec_length >= 1 && cap_in >= 1, ALM_ERR_INVALID,
                std::string(fn) + ": num_bins, rec_length and cap_in must be >= 1");
    ALM_REQUIRE(count && offset && pts && polys && rec && rec_prob && source_in && n_inst && pt && poly && whole_rec &&
                    whole_prob && page_count && page_offset && pts_out && polys_out && rec_out && prob_out && source,
                ALM_ERR_INVALID, std::string(fn) + ": null argument");
    if (turns) require_turns(turns, n_pages, fn);
    const long total = prefix_total(fn, "page", count, offset, n_pages);
    long whole = 0;
    std::vector<whole_core::Page> pages(static_cast<size_t>(n_pages));
    for (int p = 0; p < n_pages; ++p) {
      ALM_REQUIRE(n_inst[p] >= 0 && n_inst[p] <= cap_in, ALM_ERR_INVALID,
                  std::string(fn) + ": page " + std::to_string(p) + ": n_inst outside [0, cap_in]");
      whole += n_inst[p];
      pages[static_cast<size_t>(p)] = whole_core::Page{heights[p], widths[p], turns ? turns[p] : 0};
    }
    ALM_REQUIRE(total + static_cast<long>(n_pages) * cap_in <= INT_MAX / 32, ALM_ERR_INVALID,
                std::string(fn) + ": too many rows");
    ALM_REQUIRE(cap >= total + whole, ALM_ERR_INVALID,
                std::string(fn) + ": output capacity below the tile rows plus the whole-page instances");
    whole_merge(&h->c, pages, tile, overlap, num_bins, margin, rec_length, count, offset, pts, polys, rec, rec_prob,
                source_in, cap_in, n_inst, pt, poly, whole_rec, whole_prob,
                MergeRows{page_count, page_offset, pts_out, polys_out, rec_out, prob_out, source});
  });
}

int alm_omni_char_boxes(alm_ctx* h, long n_words, int rec_length, const double* polys, const int64_t* rec,
                        const float* loc, const int32_t* frame_index, int n_frames, const int32_t* frames,
                        int recog_pad_index, int rec_eos_index, int32_t* n_chars, int32_t* step, double* centre,
                        double* cov, double* box) {
  return guarded(h, [&] {
    const char* fn = "alm_omni_char_boxes";
    ALM_REQUIRE(n_words >= 0 && rec_length >= 1 && rec_length <= rec_box_core::kMaxSteps, ALM_ERR_INVALID,
                std::string(fn) + ": n_words must be >= 0 and rec_length in 1.." +
                    std::to_string(rec_box_core::kMaxSteps));
    if (n_words == 0) return;
    ALM_REQUIRE(polys && rec && loc && frame_index && frames && n_chars && step && centre && cov && box,
                ALM_ERR_INVALID, std::string(fn) + ": null argument");
    ALM_REQUIRE(n_frames >= 1, ALM_ERR_INVALID, std::string(fn) + ": words need at least one frame");
    std::vector<rec_box_core::Frame> fr(static_cast<size_t>(n_frames));
    for (int k = 0; k < n_frames; ++k) {
      const int32_t* v = frames + 7L * k;
      fr[static_cast<size_t>(k)] = rec_box_core::Frame{v[0], v[1], v[2], v[3], v[4], v[5], v[6]};
      ALM_REQUIRE(rec_box_core::valid_frame(fr[static_cast<size_t>(k)]), ALM_ERR_INVALID,
                  std::string(fn) + ": frame " + std::to_string(k) +
                      ": need positive sizes, a turn in 0..3 and the tile inside its turned page");
    }
    for (long n = 0; n < n_words; ++n)
      ALM_REQUIRE(frame_index[n] >= 0 && frame_index[n] < n_frames, ALM_ERR_INVALID,
                  std::string(fn) + ": word " + std::to_string(n) + ": frame index out of range");
    char_boxes(&h->c, n_words, rec_length, n_frames, fr.data(), frame_index, polys, rec, loc, recog_pad_index,
               rec_eos_index, n_chars, step, centre, cov, box);
  });
}

int alm_omni_select_regions(alm_ctx* h, long n_regions, int n_cand, const int32_t* frame_index, int n_frames,
                            const int32_t* frames, const int64_t* pt, const int64_t* poly, const int64_t* rec,
                            const float* rec_prob, int rec_length, int num_bins, int recog_pad_index, int rec_eos_index,
                            int32_t* kept, double* scores, double* pts, double* polys) {
  return guarded(h, [&] {
    const char* fn = "alm_omni_select_regions";
    ALM_REQUIRE(n_regions >= 0 && n_cand >= 1 && n_cand <= region_turn_core::kMaxCandidates, ALM_ERR_INVALID,
                std::string(fn) + ": n_regions must be >= 0 and n_cand in 1.." +
                    std::to_string(region_turn_core::kMaxCandidates));
    ALM_REQUIRE(rec_length >= 1 && rec_length <= rec_box_core::kMaxSteps && num_bins >= 1, ALM_ERR_INVALID,
                std::string(fn) + ": rec_length must be in 1.." + std::to_string(rec_box_core::kMaxSteps) +
                    " and num_bins >= 1");
    if (n_regions == 0) return;
    ALM_REQUIRE(frame_index && frames && pt && poly && rec && rec_prob && kept && scores && pts && polys,
                ALM_ERR_INVALID, std::string(fn) + ": null argument");
    ALM_REQUIRE(n_frames >= 1, ALM_ERR_INVALID, std::string(fn) + ": regions need at least one frame");
    std::vector<rec_box_core::Frame> fr(static_cast<size_t>(n_frames));
    for (int k = 0; k < n_frames; ++k) {
      const int32_t* v = frames + 7L * k;
      fr[static_cast<size_t>(k)] = rec_box_core::Frame{v[0], v[1], v[2], v[3], v[4], v[5], v[6]};
      ALM_REQUIRE(rec_box_core::valid_frame(fr[static_cast<size_t>(k)]), ALM_ERR_INVALID,
                  std::string(fn) + ": frame " + std::to_string(k) +
                      ": need positive sizes, a turn in 0..3 and the tile inside its turned page");
    }
    for (long g = 0; g < n_regions * n_cand; ++g)
      ALM_REQUIRE(frame_index[g] >= 0 && frame_index[g] < n_frames, ALM_ERR_INVALID,
                  std::string(fn) + ": region " + std::to_string(g / n_cand) + ", candidate " +
                      std::to_string(g % n_cand) + ": frame index out of range");
    region_select(&h->c, n_regions, n_cand, rec_length, n_frames, fr.data(), frame_index, pt, poly, rec, rec_prob,
                  num_bins, recog_pad_index, rec_eos_index, kept, scores, pts, polys);
  });
}

namespace {

// The entity table of n KIE readings (alm_omni_merge_kie_tiles: one per tile; alm_omni_merge_kie_whole_page: one per
// page): max_ent slots per reading, n_ent used, and the totals of entities and of their words
struct EntityTable {
  std::vector<kie_tile_core::Entity> table;
  std::vector<int> n_ent;
  int max_ent = 1;
  long ents = 0, words = 0;
};

// The walk of every reading's token stream: the checks (the refusals name each reading `what` and its index), and the
// entity table of the merge
EntityTable walk_readings(const char* fn, const char* what, int n, const int32_t* n_tok, const int64_t* tokens,
                          const float* tok_prob, int max_tok, const int32_t* n_inst, const int32_t* inst_pos,
                          int max_inst, int num_bins, int class_base, int n_classes) {
  EntityTable t;
  std::vector<std::vector<kie_tile_core::Entity>> per(static_cast<size_t>(n));
  t.n_ent.resize(static_cast<size_t>(n));
  for (int k = 0; k < n; ++k) {
    const std::string at = std::string(fn) + ": " + what + " " + std::to_string(k);
    ALM_REQUIRE(n_tok[k] >= 0 && n_tok[k] <= max_tok, ALM_ERR_INVALID, at + ": n_tok outside [0, max_tok]");
    ALM_REQUIRE(n_inst[k] >= 0 && n_inst[k] <= max_inst, ALM_ERR_INVALID, at + ": n_inst outside [0, max_inst]");
    const long o = static_cast<long>(k) * max_tok;
    int pairs = 0;
    const int st = kie_tile_core::walk(tokens + o, tok_prob + o, n_tok[k], inst_pos + static_cast<long>(k) * max_inst,
                                       n_inst[k], num_bins, class_base, n_classes, &per[static_cast<size_t>(k)], &pairs);
    ALM_REQUIRE(st != kie_tile_core::kWalkBadClass, ALM_ERR_INVALID, at + ": a token is neither a bin nor an entity class");
    ALM_REQUIRE(st == kie_tile_core::kWalkOk && pairs == n_inst[k], ALM_ERR_INVALID,
                at + ": inst_pos does not match the (x, y) pairs of the token stream");
    t.n_ent[static_cast<size_t>(k)] = static_cast<int>(per[static_cast<size_t>(k)].size());
    t.max_ent = std::max(t.max_ent, t.n_ent[static_cast<size_t>(k)]);
    t.ents += t.n_ent[static_cast<size_t>(k)];
    for (const kie_tile_core::Entity& e : per[static_cast<size_t>(k)]) t.words += e.words;
  }
  t.table.assign(static_cast<size_t>(n) * t.max_ent, kie_tile_core::Entity{0, 0.f, 0, 0});
  for (int k = 0; k < n; ++k)
    std::copy(per[static_cast<size_t>(k)].begin(), per[static_cast<size_t>(k)].end(),
              t.table.begin() + static_cast<long>(k) * t.max_ent);
  return t;
}

// The output capacities and buffers of a KIE merge that may keep `ents` entities with `words` words
void require_kie_out(const char* fn, long ents, long words, long cap_ent, long cap_words, const void* ent_class,
                     const void* ent_prob, const void* word_offset, const void* word_count, const void* ent_source,
                     const void* word_rect, const void* word_poly, const void* word_source) {
  ALM_REQUIRE(cap_ent >= ents && cap_words >= words, ALM_ERR_INVALID,
              std::string(fn) + ": output capacity below the entities (cap_ent) or their words (cap_words)");
  ALM_REQUIRE(ents == 0 || (ent_class && ent_prob && word_offset && word_count && ent_source), ALM_ERR_INVALID,
              std::string(fn) + ": null entity output buffer");
  ALM_REQUIRE(words == 0 || (word_rect && word_poly && word_source), ALM_ERR_INVALID,
              std::string(fn) + ": null word output buffer");
}

}  // namespace

int alm_omni_merge_kie_tiles(alm_ctx* h, const int* heights, const int* widths, int n_pages, const int32_t* turns,
                             int tile, int overlap, int n_tiles, const int* tile_page, const int* tile_origin,
                             const int32_t* n_tok, const int64_t* tokens, const float* tok_prob, int max_tok,
                             const int32_t* n_inst, const int32_t* inst_pos, const int64_t* poly, int max_inst,
                             int num_bins, int class_base, int n_classes, double margin, double band, double iou,
                             int32_t* page_count, int32_t* page_offset, int32_t* ent_class, float* ent_prob,
                             int32_t* word_offset, int32_t* word_count, int32_t* ent_source, long cap_ent,
                             double* word_rect, double* word_poly, int32_t* word_source, long cap_words) {
  return guarded(h, [&] {
    const char* fn = "alm_omni_merge_kie_tiles";
    ALM_REQUIRE(max_tok >= 1 && max_inst >= 1 && num_bins >= 1 && n_classes >= 1, ALM_ERR_INVALID,
                std::string(fn) + ": max_tok, max_inst, num_bins and n_classes must be >= 1");
    ALM_REQUIRE(n_tok && tokens && tok_prob && n_inst && inst_pos && poly && page_count && page_offset, ALM_ERR_INVALID,
                std::string(fn) + ": null argument");
    const std::vector<tile_core::Tile> tiles = merge_plan(fn, heights, widths, n_pages, turns, tile, overlap, margin,
                                                          band, iou, n_tiles, tile_page, tile_origin);
    const EntityTable t = walk_readings(fn, "tile", n_tiles, n_tok, tokens, tok_prob, max_tok, n_inst, inst_pos,
                                        max_inst, num_bins, class_base, n_classes);
    ALM_REQUIRE(static_cast<long>(n_tiles) * t.max_ent + t.words <= INT_MAX / 32, ALM_ERR_INVALID,
                std::string(fn) + ": too many entities or words");
    require_kie_out(fn, t.ents, t.words, cap_ent, cap_words, ent_class, ent_prob, word_offset, word_count, ent_source,
                    word_rect, word_poly, word_source);
    kie_merge(&h->c, tiles, n_pages, t.max_ent, t.n_ent.data(), t.table.data(), max_inst, poly, num_bins, margin, iou,
              page_count, page_offset, ent_class, ent_prob, word_offset, word_count, ent_source, word_rect, word_poly,
              word_source);
  });
}

int alm_omni_merge_kie_whole_page(alm_ctx* h, const int* heights, const int* widths, int n_pages, const int32_t* turns,
                                  int tile, int overlap, double margin, int num_bins, int class_base, int n_classes,
                                  const int32_t* count, const int32_t* offset, const int32_t* ent_class,
                                  const float* ent_prob, const int32_t* word_offset, const int32_t* word_count,
                                  const int32_t* ent_source, const double* word_rect, const double* word_poly,
                                  const int32_t* word_source, const int32_t* n_tok, const int64_t* tokens,
                                  const float* tok_prob, int max_tok, const int32_t* n_inst, const int32_t* inst_pos,
                                  const int64_t* poly, int max_inst, int32_t* page_count, int32_t* page_offset,
                                  int32_t* ent_class_out, float* ent_prob_out, int32_t* word_offset_out,
                                  int32_t* word_count_out, int32_t* ent_source_out, long cap_ent,
                                  double* word_rect_out, double* word_poly_out, int32_t* word_source_out,
                                  long cap_words) {
  return guarded(h, [&] {
    const char* fn = "alm_omni_merge_kie_whole_page";
    ALM_REQUIRE(pages_ok(heights, widths, n_pages) && tile_core::valid_layout(tile, overlap), ALM_ERR_INVALID,
                std::string(fn) + ": page sizes, or tile size / overlap (need tile >= 64, 0 <= 2 overlap <= tile)");
    ALM_REQUIRE(std::isfinite(margin) && margin >= 0.0, ALM_ERR_INVALID,
                std::string(fn) + ": margin must be finite and >= 0");
    ALM_REQUIRE(max_tok >= 1 && max_inst >= 1 && num_bins >= 1 && n_classes >= 1, ALM_ERR_INVALID,
                std::string(fn) + ": max_tok, max_inst, num_bins and n_classes must be >= 1");
    ALM_REQUIRE(count && offset && n_tok && tokens && tok_prob && n_inst && inst_pos && poly && page_count &&
                    page_offset,
                ALM_ERR_INVALID, std::string(fn) + ": null argument");
    if (turns) require_turns(turns, n_pages, fn);
    // the tile entities: page rows, then each entity's word rows, both exclusive prefixes of their counts
    const long E = prefix_total(fn, "page", count, offset, n_pages);
    ALM_REQUIRE(E == 0 || (ent_class && ent_prob && word_offset && word_count && ent_source), ALM_ERR_INVALID,
                std::string(fn) + ": null tile entity buffer");
    ALM_REQUIRE(E <= INT_MAX / 32, ALM_ERR_INVALID, std::string(fn) + ": too many entities");
    const long W = E ? prefix_total(fn, "entity", word_count, word_offset, E) : 0;
    ALM_REQUIRE(W == 0 || (word_rect && word_poly && word_source), ALM_ERR_INVALID,
                std::string(fn) + ": null tile word buffer");
    const EntityTable t = walk_readings(fn, "page", n_pages, n_tok, tokens, tok_prob, max_tok, n_inst, inst_pos,
                                        max_inst, num_bins, class_base, n_classes);
    ALM_REQUIRE(E + static_cast<long>(n_pages) * t.max_ent + W + t.words <= INT_MAX / 32, ALM_ERR_INVALID,
                std::string(fn) + ": too many entities or words");
    require_kie_out(fn, E + t.ents, W + t.words, cap_ent, cap_words, ent_class_out, ent_prob_out, word_offset_out,
                    word_count_out, ent_source_out, word_rect_out, word_poly_out, word_source_out);
    std::vector<tile_core::Tile> wt(static_cast<size_t>(n_pages));
    for (int p = 0; p < n_pages; ++p)
      wt[static_cast<size_t>(p)] = kie_whole_core::whole_tile(p, heights[p], widths[p], turns ? turns[p] : 0);
    kie_whole_merge(&h->c, wt, tile, overlap, num_bins, margin, count, offset, ent_class, ent_prob, word_offset,
                    word_count, ent_source, word_rect, word_poly, word_source, t.max_ent, t.n_ent.data(),
                    t.table.data(), max_inst, poly, page_count, page_offset, ent_class_out, ent_prob_out,
                    word_offset_out, word_count_out, ent_source_out, word_rect_out, word_poly_out, word_source_out);
  });
}

int alm_omni_group_lines(alm_ctx* h, int n_pages, const int* page_count, const int* page_offset, const double* polys,
                         double cos_tol, double height_ratio, double max_offset, double max_overlap, double max_gap,
                         int* n_lines, int* line_offset, int* line_first, int* line_words, int32_t* order,
                         int32_t* line_of, int32_t* rank_of, double* line_polys, long cap) {
  return guarded(h, [&] {
    const std::string fn = "alm_omni_group_lines: ";
    ALM_REQUIRE(n_pages >= 1, ALM_ERR_INVALID, fn + "n_pages must be >= 1");
    ALM_REQUIRE(page_count != nullptr, ALM_ERR_INVALID, fn + "page_count is null");
    ALM_REQUIRE(page_offset != nullptr, ALM_ERR_INVALID, fn + "page_offset is null");
    long N = 0;
    for (int p = 0; p < n_pages; ++p) {
      ALM_REQUIRE(page_count[p] >= 0, ALM_ERR_INVALID, fn + "page_count[" + std::to_string(p) + "] is negative");
      N += page_count[p];
    }
    ALM_REQUIRE(N <= INT_MAX / 8, ALM_ERR_INVALID, fn + "page_count: too many words");
    std::vector<std::pair<int, int>> rows;  // (first row, count) of the pages that have words
    for (int p = 0; p < n_pages; ++p) {
      ALM_REQUIRE(page_offset[p] >= 0 && static_cast<long>(page_offset[p]) + page_count[p] <= N, ALM_ERR_INVALID,
                  fn + "page_offset[" + std::to_string(p) + "]: the page's rows leave [0, sum of page_count)");
      if (page_count[p] > 0) rows.emplace_back(page_offset[p], page_count[p]);
    }
    std::sort(rows.begin(), rows.end());
    for (size_t k = 1; k < rows.size(); ++k)
      ALM_REQUIRE(rows[k - 1].first + rows[k - 1].second <= rows[k].first, ALM_ERR_INVALID,
                  fn + "page_offset: the rows of two pages overlap");
    const group_core::Params prm{cos_tol, height_ratio, max_offset, max_overlap, max_gap};
    ALM_REQUIRE(cos_tol >= -1.0 && cos_tol <= 1.0, ALM_ERR_INVALID, fn + "cos_tol must be in [-1, 1]");
    ALM_REQUIRE(height_ratio >= 0.0 && height_ratio <= 1.0, ALM_ERR_INVALID, fn + "height_ratio must be in [0, 1]");
    ALM_REQUIRE(std::isfinite(max_offset) && max_offset >= 0.0, ALM_ERR_INVALID, fn + "max_offset must be finite and >= 0");
    ALM_REQUIRE(std::isfinite(max_overlap) && max_overlap >= 0.0, ALM_ERR_INVALID,
                fn + "max_overlap must be finite and >= 0");
    ALM_REQUIRE(std::isfinite(max_gap) && max_gap >= 0.0, ALM_ERR_INVALID, fn + "max_gap must be finite and >= 0");
    ALM_REQUIRE(cap >= N, ALM_ERR_INVALID, fn + "cap is below the number of words");
    ALM_REQUIRE(n_lines != nullptr, ALM_ERR_INVALID, fn + "n_lines is null");
    ALM_REQUIRE(line_offset != nullptr, ALM_ERR_INVALID, fn + "line_offset is null");
    if (N > 0) {
      ALM_REQUIRE(polys != nullptr, ALM_ERR_INVALID, fn + "polys is null");
      ALM_REQUIRE(line_first != nullptr, ALM_ERR_INVALID, fn + "line_first is null");
      ALM_REQUIRE(line_words != nullptr, ALM_ERR_INVALID, fn + "line_words is null");
      ALM_REQUIRE(order != nullptr, ALM_ERR_INVALID, fn + "order is null");
      ALM_REQUIRE(line_of != nullptr, ALM_ERR_INVALID, fn + "line_of is null");
      ALM_REQUIRE(rank_of != nullptr, ALM_ERR_INVALID, fn + "rank_of is null");
      ALM_REQUIRE(line_polys != nullptr, ALM_ERR_INVALID, fn + "line_polys is null");
    }
    group_lines(&h->c, n_pages, page_count, page_offset, N, polys, prm, n_lines, line_offset, line_first, line_words,
                order, line_of, rank_of, line_polys);
  });
}

// ------------------------------------------------------------------------------------------ OmniParser
int alm_omni_encode(alm_ctx* h, const float* img, const uint8_t* mask, int B, int H, int W) {
  return guarded(h, [&] {
    ALM_REQUIRE(img != nullptr && B > 0 && H > 0 && W > 0, ALM_ERR_INVALID, "alm_omni_encode arguments");
    const size_t px = static_cast<size_t>(B) * H * W;
    const float* dimg = static_cast<const float*>(stage_input(h, img, px * 3 * sizeof(float), &h->dev_in, &h->dev_in_bytes));
    const uint8_t* dmask = static_cast<const uint8_t*>(stage_input(h, mask, px, &h->dev_mask, &h->dev_mask_bytes));
    omni_encode(&h->c, dimg, dmask, B, H, W);
  });
}

int alm_omni_encode_pages(alm_ctx* h, const float* img, int B, int Hc, int Wc, const int* heights, const int* widths) {
  return guarded(h, [&] {
    ALM_REQUIRE(img != nullptr && heights != nullptr && widths != nullptr && B > 0 && Hc > 0 && Wc > 0, ALM_ERR_INVALID,
                "alm_omni_encode_pages arguments");
    for (int b = 0; b < B; ++b)
      ALM_REQUIRE(heights[b] >= 32 && widths[b] >= 32 && heights[b] <= Hc && widths[b] <= Wc, ALM_ERR_INVALID,
                  "alm_omni_encode_pages: page " + std::to_string(b) + " must be at least 32x32 and fit the canvas");
    ALM_REQUIRE(h->c.omni != nullptr, ALM_ERR_STATE, "alm_omni_encode_pages before alm_load_weights");
    const size_t px = static_cast<size_t>(B) * Hc * Wc;
    const float* dimg = static_cast<const float*>(stage_input(h, img, px * 3 * sizeof(float), &h->dev_in, &h->dev_in_bytes));
    omni_encode_pages(&h->c, dimg, B, Hc, Wc, heights, widths);
  });
}

int alm_omni_page_shapes(alm_ctx* h, int* mh, int* mw) {
  return guarded(h, [&] {
    const OmniModel* m = h->c.omni;
    ALM_REQUIRE(m && m->encoded, ALM_ERR_STATE, "no encoded batch");
    ALM_REQUIRE(mh && mw, ALM_ERR_INVALID, "alm_omni_page_shapes arguments");
    std::copy(m->page_mh.begin(), m->page_mh.end(), mh);
    std::copy(m->page_mw.begin(), m->page_mw.end(), mw);
  });
}

int alm_omni_memory_shape(alm_ctx* h, int* B, int* mh, int* mw) {
  return guarded(h, [&] {
    ALM_REQUIRE(h->c.omni && h->c.omni->encoded, ALM_ERR_STATE, "no encoded batch");
    ALM_REQUIRE(!h->c.omni->mixed, ALM_ERR_STATE, "pages of different sizes have no common grid: use alm_omni_page_shapes");
    if (B) *B = h->c.omni->B;
    if (mh) *mh = h->c.omni->mh;
    if (mw) *mw = h->c.omni->mw;
  });
}

int alm_omni_last_timing(alm_ctx* h, float* encode_ms, float* pt_ms, float* polyrec_ms) {
  return guarded(h, [&] {
    ALM_CHECK_CUDA(cudaStreamSynchronize(h->c.stream));
    float e = -1.f, p = -1.f, r = -1.f;
    if (h->c.timing_valid[0]) ALM_CHECK_CUDA(cudaEventElapsedTime(&e, h->c.ev_t[0], h->c.ev_t[1]));
    if (h->c.timing_valid[1]) {
      ALM_CHECK_CUDA(cudaEventElapsedTime(&p, h->c.ev_t[2], h->c.ev_t[3]));
      ALM_CHECK_CUDA(cudaEventElapsedTime(&r, h->c.ev_t[3], h->c.ev_t[4]));
    }
    if (encode_ms) *encode_ms = e;
    if (pt_ms) *pt_ms = p;
    if (polyrec_ms) *polyrec_ms = r;
  });
}

int alm_omni_vocab(alm_ctx* h) { return (h && h->c.omni) ? h->c.omni->V : ALM_ERR_STATE; }

int alm_omni_get_feature(alm_ctx* h, int level, float* out, size_t out_elems) {
  return guarded(h, [&] {
    OmniModel* m = h->c.omni;
    ALM_REQUIRE(m && m->encoded, ALM_ERR_STATE, "no encoded batch");
    ALM_REQUIRE(!m->mixed, ALM_ERR_UNSUPPORTED, "stage features are not kept for pages of different sizes");
    ALM_REQUIRE(level >= 0 && level < 4 && out, ALM_ERR_INVALID, "feature level");
    const size_t n = static_cast<size_t>(m->B) * m->Hs[level] * m->Ws[level] * (128 << level);
    ALM_REQUIRE(out_elems == n, ALM_ERR_INVALID, "feature buffer size mismatch: expected " + std::to_string(n));
    d2h(&h->c, out, m->feat[level], n * sizeof(float));
    ALM_CHECK_CUDA(cudaStreamSynchronize(h->c.stream));
  });
}

int alm_omni_get_memory(alm_ctx* h, int which, float* out, size_t out_elems) {
  return guarded(h, [&] {
    OmniModel* m = h->c.omni;
    ALM_REQUIRE(m && m->encoded, ALM_ERR_STATE, "no encoded batch");
    const size_t n = static_cast<size_t>(m->B) * m->M * 512;
    ALM_REQUIRE(out && out_elems == n && (which == 0 || which == 1), ALM_ERR_INVALID, "memory buffer size mismatch");
    d2h(&h->c, out, which == 0 ? m->memory : m->pos, n * sizeof(float));
    ALM_CHECK_CUDA(cudaStreamSynchronize(h->c.stream));
  });
}

int alm_omni_decode(alm_ctx* h, const int64_t* pt_prompt, int n_prompt, const alm_decode_cfg* cfg, int32_t* n_inst,
                    int64_t* pt, int64_t* poly, int64_t* rec, float* rec_prob) {
  return guarded(h, [&] {
    ALM_REQUIRE(pt_prompt && cfg && n_inst && pt && poly && rec && rec_prob, ALM_ERR_INVALID, "null argument");
    omni_decode(&h->c, pt_prompt, n_prompt, *cfg, n_inst, pt, poly, rec, rec_prob);
  });
}

int alm_omni_decode_prompts(alm_ctx* h, const int64_t* prompts, int P, int n_prompt, const alm_decode_cfg* cfg,
                            int32_t* n_inst, int64_t* pt, int64_t* poly, int64_t* rec, float* rec_prob) {
  return guarded(h, [&] {
    ALM_REQUIRE(prompts && cfg && n_inst && pt && poly && rec && rec_prob, ALM_ERR_INVALID, "null argument");
    omni_decode_prompts(&h->c, prompts, P, n_prompt, *cfg, n_inst, pt, poly, rec, rec_prob);
  });
}

int alm_omni_decode_dense(alm_ctx* h, const int64_t* pt_prompt, int n_prompt, const alm_decode_cfg* cfg, int nx, int ny,
                          double iou, int cap, int32_t* n_inst, int64_t* pt, int64_t* poly, int64_t* rec,
                          float* rec_prob, int32_t* window, int32_t* grid, uint8_t* saturated) {
  return guarded(h, [&] {
    ALM_REQUIRE(pt_prompt && cfg && n_inst && pt && poly && rec && rec_prob && window && grid && saturated,
                ALM_ERR_INVALID, "alm_omni_decode_dense: null argument");
    omni_decode_dense(&h->c, pt_prompt, n_prompt, *cfg, nx, ny, iou, cap, n_inst, pt, poly, rec, rec_prob, window, grid,
                      saturated);
  });
}

int alm_omni_get_dense_loops(alm_ctx* h, int32_t* out, size_t elems, int32_t* n_loops) {
  return guarded(h, [&] {
    ALM_REQUIRE(n_loops, ALM_ERR_INVALID, "alm_omni_get_dense_loops: null argument");
    *n_loops = static_cast<int32_t>(omni_dense_loops(&h->c, out, elems));
  });
}

int alm_omni_decode_kie(alm_ctx* h, const int64_t* pt_prompt, int n_prompt, const alm_decode_cfg* cfg, int32_t* n_tok,
                        int64_t* pt_tokens, float* pt_probs, int32_t* n_inst, int32_t* inst_pos, int64_t* poly,
                        int64_t* rec, float* rec_prob) {
  return guarded(h, [&] {
    ALM_REQUIRE(pt_prompt && cfg && n_tok && pt_tokens && pt_probs && n_inst && inst_pos && poly && rec && rec_prob,
                ALM_ERR_INVALID, "null argument");
    omni_decode_kie(&h->c, pt_prompt, n_prompt, *cfg, n_tok, pt_tokens, pt_probs, n_inst, inst_pos, poly, rec, rec_prob);
  });
}

int alm_omni_decode_points(alm_ctx* h, const int64_t* pt_prompt, int n_prompt, const alm_decode_cfg* cfg, int32_t* n_tok,
                           int64_t* pt_tokens, float* pt_probs) {
  return guarded(h, [&] {
    ALM_REQUIRE(pt_prompt && cfg && n_tok && pt_tokens, ALM_ERR_INVALID, "null argument");
    omni_decode_points(&h->c, pt_prompt, n_prompt, *cfg, n_tok, pt_tokens, pt_probs);
  });
}

int alm_omni_decode_at(alm_ctx* h, const int32_t* xy, const int32_t* count, int cap, const alm_decode_cfg* cfg,
                       int64_t* poly, int64_t* rec, float* rec_prob) {
  return guarded(h, [&] {
    ALM_REQUIRE(xy && count && cfg && poly && rec && rec_prob, ALM_ERR_INVALID, "null argument");
    omni_decode_at(&h->c, xy, count, cap, *cfg, poly, rec, rec_prob);
  });
}

int alm_omni_set_rec_candidates(alm_ctx* h, int k) {
  return guarded(h, [&] {
    ALM_REQUIRE(k >= 0 && k <= ALM_MAX_CANDIDATES, ALM_ERR_INVALID, "alm_omni_set_rec_candidates: k must be 0..8");
    ALM_REQUIRE(k == 0 || h->c.rec_beams == 0, ALM_ERR_INVALID,
                "alm_omni_set_rec_candidates: candidates cannot be combined with beams (set W = 0 first)");
    h->c.rec_topk = k;
  });
}

int alm_omni_set_rec_beams(alm_ctx* h, int W, float length_penalty) {
  return guarded(h, [&] {
    ALM_REQUIRE(W >= 0 && W <= ALM_MAX_BEAMS, ALM_ERR_INVALID, "alm_omni_set_rec_beams: W must be 0..8");
    ALM_REQUIRE(length_penalty >= 0.f && length_penalty <= 2.f, ALM_ERR_INVALID,
                "alm_omni_set_rec_beams: length_penalty must be in [0, 2]");
    ALM_REQUIRE(W == 0 || h->c.rec_topk == 0, ALM_ERR_INVALID,
                "alm_omni_set_rec_beams: beams cannot be combined with candidates (set k = 0 first)");
    ALM_REQUIRE(W == 0 || !h->c.rec_locations, ALM_ERR_INVALID,
                "alm_omni_set_rec_beams: beams cannot be combined with character locations (turn them off first)");
    h->c.rec_beams = W;
    h->c.beam_alpha = length_penalty;
  });
}

int alm_omni_get_rec_beams(alm_ctx* h, int64_t* ids, float* probs, float* scores, size_t elems) {
  return guarded(h, [&] {
    ALM_REQUIRE(ids && probs && scores, ALM_ERR_INVALID, "null argument");
    omni_rec_beams(&h->c, ids, probs, scores, elems);
  });
}

int alm_omni_set_rec_locations(alm_ctx* h, int on) {
  return guarded(h, [&] {
    ALM_REQUIRE(!on || h->c.rec_beams == 0, ALM_ERR_INVALID,
                "alm_omni_set_rec_locations: character locations cannot be combined with beams (set W = 0 first)");
    h->c.rec_locations = on != 0;
  });
}

int alm_omni_set_rec_charset(alm_ctx* h, const uint8_t* allowed, int n_sets, int n_chars, const int32_t* row_set,
                             size_t n_rows) {
  return guarded(h, [&] {
    const std::string fn = "alm_omni_set_rec_charset: ";
    ALM_REQUIRE(n_sets >= 0 && n_sets <= ALM_MAX_CHARSETS, ALM_ERR_INVALID,
                fn + "n_sets must be 0.." + std::to_string(ALM_MAX_CHARSETS));
    Ctx& c = h->c;
    if (n_sets == 0) {  // off: the default, nothing allocated or launched
      c.rec_cs_sets = c.rec_cs_chars = 0;
      c.rec_cs_allowed.clear();
      c.rec_cs_rows.clear();
      return;
    }
    ALM_REQUIRE(allowed != nullptr && n_chars >= 1, ALM_ERR_INVALID, fn + "allowed must be [n_sets][n_chars], n_chars >= 1");
    ALM_REQUIRE((row_set == nullptr) == (n_rows == 0), ALM_ERR_INVALID, fn + "row_set and n_rows go together");
    const size_t n = static_cast<size_t>(n_sets) * n_chars;
    for (int k = 0; k < n_sets; ++k)
      ALM_REQUIRE(std::any_of(allowed + static_cast<size_t>(k) * n_chars, allowed + (k + 1) * static_cast<size_t>(n_chars),
                              [](uint8_t v) { return v != 0; }),
                  ALM_ERR_INVALID, fn + "set " + std::to_string(k) + " is empty");
    for (size_t r = 0; r < n_rows; ++r)
      ALM_REQUIRE(row_set[r] >= 0 && row_set[r] < n_sets, ALM_ERR_INVALID,
                  fn + "row " + std::to_string(r) + "'s set index is outside [0, n_sets)");
    c.rec_cs_allowed.resize(n);
    for (size_t i = 0; i < n; ++i) c.rec_cs_allowed[i] = allowed[i] != 0;
    c.rec_cs_rows.assign(row_set, row_set + n_rows);
    c.rec_cs_sets = n_sets;
    c.rec_cs_chars = n_chars;
  });
}

int alm_omni_get_rec_locations(alm_ctx* h, float* out, size_t elems) {
  return guarded(h, [&] {
    ALM_REQUIRE(out, ALM_ERR_INVALID, "null argument");
    omni_rec_locations(&h->c, out, elems);
  });
}

int alm_omni_get_rec_candidates(alm_ctx* h, int64_t* ids, float* probs, size_t elems) {
  return guarded(h, [&] {
    ALM_REQUIRE(ids && probs, ALM_ERR_INVALID, "null argument");
    omni_rec_candidates(&h->c, ids, probs, elems);
  });
}

int alm_omni_decode_logits(alm_ctx* h, int image, int kind, const int64_t* seq, int n_seq, int len, float* logits) {
  return guarded(h, [&] {
    ALM_REQUIRE(seq && logits, ALM_ERR_INVALID, "null argument");
    omni_decode_logits(&h->c, image, kind, seq, n_seq, len, logits);
  });
}

// ------------------------------------------------------------------------------------------ MGP-STR
namespace {

// the caller's [B][3][32][128] crop batch on the device
const float* stage_crops(alm_ctx* h, const float* img, int B) {
  return static_cast<const float*>(
      stage_input(h, img, static_cast<size_t>(B) * 3 * 32 * 128 * sizeof(float), &h->dev_in, &h->dev_in_bytes));
}

// one attention-map plane per A^3 head of the loaded checkpoint
void require_a3_heads(alm_ctx* h, int n_heads, const char* fn) {
  int n_a3 = 0;
  mgp_info(h->c.mgp, nullptr, nullptr, nullptr, &n_a3, nullptr);
  ALM_REQUIRE(n_heads == n_a3, ALM_ERR_INVALID,
              std::string(fn) + ": " + std::to_string(n_heads) + " head planes, but the checkpoint has " +
                  std::to_string(n_a3) + " A^3 heads");
}

// the page geometry of R quad (9 values each) or curve (16 values each) regions, with their crop sizes
std::vector<box_core::BoxGeom> region_geom(int kind, int R, const int* sizes, const double* geom, const char* fn) {
  const int nv = kind == ALM_BOX_QUAD ? 9 : 16;
  std::vector<box_core::BoxGeom> g(static_cast<size_t>(R));
  for (int r = 0; r < R; ++r) {
    box_core::BoxGeom& d = g[static_cast<size_t>(r)];
    d.cw = sizes[2L * r];
    d.ch = sizes[2L * r + 1];
    ALM_REQUIRE(d.cw >= 1 && d.ch >= 1, ALM_ERR_INVALID,
                std::string(fn) + ": region " + std::to_string(r) + ": crop size");
    for (int i = 0; i < nv; ++i) {
      d.g[i] = geom[static_cast<long>(nv) * r + i];
      ALM_REQUIRE(isfinite(d.g[i]), ALM_ERR_INVALID,
                  std::string(fn) + ": region " + std::to_string(r) + ": non-finite geometry");
    }
  }
  return g;
}

}  // namespace

int alm_mgpstr_forward(alm_ctx* h, const float* img, int B, float* attn, float* char_logits, float* bpe_logits,
                       float* wp_logits, int32_t* ids, float* prob) {
  return guarded(h, [&] {
    ALM_REQUIRE(img && B > 0, ALM_ERR_INVALID, "alm_mgpstr_forward arguments");
    mgp_forward(&h->c, stage_crops(h, img, B), B, attn, char_logits, bpe_logits, wp_logits, ids, prob);
  });
}

int alm_mgpstr_topk(alm_ctx* h, const float* img, int B, int k, int32_t* ids, float* probs) {
  return guarded(h, [&] {
    ALM_REQUIRE(img && B > 0 && ids && probs, ALM_ERR_INVALID, "alm_mgpstr_topk arguments");
    ALM_REQUIRE(k >= 1 && k <= ALM_MAX_CANDIDATES, ALM_ERR_INVALID, "alm_mgpstr_topk: k must be 1..8");
    ALM_REQUIRE(h->c.mgp != nullptr, ALM_ERR_STATE, "alm_mgpstr_topk needs an MGP-STR checkpoint in this context");
    mgp_forward(&h->c, stage_crops(h, img, B), B, nullptr, nullptr, nullptr, nullptr, ids, probs, k);
  });
}

int alm_mgpstr_forward_boxes(alm_ctx* h, const float* img, int B, int k, int geom_kind, int n_geom, const int* sizes,
                             const double* geom, int n_heads, int32_t* ids, float* probs, int32_t* n, float* boxes,
                             float* centres) {
  return guarded(h, [&] {
    ALM_REQUIRE(img && B > 0 && ids && probs && n && boxes && centres, ALM_ERR_INVALID,
                "alm_mgpstr_forward_boxes arguments");
    ALM_REQUIRE(k >= 0 && k <= ALM_MAX_CANDIDATES, ALM_ERR_INVALID, "alm_mgpstr_forward_boxes: k must be 0..8");
    ALM_REQUIRE(h->c.mgp != nullptr, ALM_ERR_STATE, "alm_mgpstr_forward_boxes needs an MGP-STR checkpoint in this context");
    require_a3_heads(h, n_heads, "alm_mgpstr_forward_boxes");
    ALM_REQUIRE(geom_kind == ALM_BOX_CROP || geom_kind == ALM_BOX_QUAD || geom_kind == ALM_BOX_CURVE, ALM_ERR_INVALID,
                "alm_mgpstr_forward_boxes: geom_kind must be 0 (crop), 1 (quad) or 2 (curve)");
    ALM_REQUIRE(n_geom == B, ALM_ERR_INVALID,
                "alm_mgpstr_forward_boxes: geometry of " + std::to_string(n_geom) + " regions for " + std::to_string(B) +
                    " crops");
    std::vector<box_core::BoxGeom> g;
    if (geom_kind != ALM_BOX_CROP) {
      ALM_REQUIRE(sizes && geom, ALM_ERR_INVALID, "alm_mgpstr_forward_boxes: quad / curve geometry needs sizes and geom");
      g = region_geom(geom_kind, B, sizes, geom, "alm_mgpstr_forward_boxes");
    }
    const MgpBoxes mb{geom_kind, g.empty() ? nullptr : g.data(), n, boxes, centres};
    mgp_forward(&h->c, stage_crops(h, img, B), B, nullptr, nullptr, nullptr, nullptr, ids, probs, k, &mb);
  });
}

int alm_mgpstr_forward_lines(alm_ctx* h, const float* img, int B, int R, const int* windows, int kind, const int* sizes,
                             const double* geom, int n_heads, int32_t* ids, float* probs, int32_t* n, float* boxes,
                             float* centres) {
  return guarded(h, [&] {
    ALM_REQUIRE(img && B > 0 && R > 0 && windows && sizes && geom && ids && probs && n && boxes && centres,
                ALM_ERR_INVALID, "alm_mgpstr_forward_lines arguments");
    ALM_REQUIRE(h->c.mgp != nullptr, ALM_ERR_STATE, "alm_mgpstr_forward_lines needs an MGP-STR checkpoint in this context");
    require_a3_heads(h, n_heads, "alm_mgpstr_forward_lines");
    ALM_REQUIRE(kind == ALM_BOX_QUAD || kind == ALM_BOX_CURVE, ALM_ERR_INVALID,
                "alm_mgpstr_forward_lines: kind must be 1 (quad) or 2 (curve)");
    const std::vector<box_core::BoxGeom> g = region_geom(kind, R, sizes, geom, "alm_mgpstr_forward_lines");
    std::vector<line_core::LineWin> win;
    std::vector<int> wstart(static_cast<size_t>(R) + 1, 0);
    for (int r = 0; r < R; ++r) {
      const line_core::Windows w = line_core::line_windows(g[static_cast<size_t>(r)].cw, g[static_cast<size_t>(r)].ch);
      ALM_REQUIRE(windows[r] == w.n, ALM_ERR_INVALID,
                  "alm_mgpstr_forward_lines: region " + std::to_string(r) + ": " + std::to_string(windows[r]) +
                      " windows, but its crop has " + std::to_string(w.n));
      ALM_REQUIRE(wstart[static_cast<size_t>(r)] + w.n <= B, ALM_ERR_INVALID,
                  "alm_mgpstr_forward_lines: the window counts exceed B = " + std::to_string(B));
      for (int i = 0; i < w.n; ++i) win.push_back(line_core::LineWin{r, w.x0[i], w.wn, 0});
      wstart[static_cast<size_t>(r) + 1] = wstart[static_cast<size_t>(r)] + w.n;
    }
    ALM_REQUIRE(wstart.back() == B, ALM_ERR_INVALID,
                "alm_mgpstr_forward_lines: the window counts sum to " + std::to_string(wstart.back()) + ", not B = " +
                    std::to_string(B));
    Ctx* c = &h->c;
    c->ensure_ws();
    ALM_REQUIRE(mgp_lines_bytes(B, R) <= c->ws.cap, ALM_ERR_INVALID,
                "alm_mgpstr_forward_lines: " + std::to_string(B) + " windows do not fit in the workspace");
    const MgpLines ml{kind, R, g.data(), win.data(), wstart.data(), ids, probs, n, boxes, centres};
    mgp_forward(c, stage_crops(h, img, B), B, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, nullptr, &ml);
  });
}

int alm_mgpstr_forward_oriented(alm_ctx* h, const float* img, int B, int N, const int32_t* turns, int R,
                                const int* readings, int k, int lines, int kind, const int* windows, const int* sizes,
                                const double* geom, int n_heads, int32_t* ids, float* probs, int32_t* n, float* boxes,
                                float* centres, int32_t* turns_out, float* conf) {
  return guarded(h, [&] {
    const char* fn = "alm_mgpstr_forward_oriented";
    const std::string f(fn);
    ALM_REQUIRE(img && B > 0 && N > 0 && R > 0 && turns && readings && ids && probs && turns_out && conf,
                ALM_ERR_INVALID, f + " arguments");
    ALM_REQUIRE(lines == 0 || lines == 1, ALM_ERR_INVALID, f + ": lines must be 0 or 1");
    ALM_REQUIRE(k >= 0 && k <= ALM_MAX_CANDIDATES && !(lines && k), ALM_ERR_INVALID,
                f + ": k must be 0..8 (0 for lines)");
    ALM_REQUIRE(h->c.mgp != nullptr, ALM_ERR_STATE, f + " needs an MGP-STR checkpoint in this context");
    require_a3_heads(h, n_heads, fn);
    require_turns(turns, N, fn);
    std::vector<int> rstart(static_cast<size_t>(R) + 1, 0);
    for (int r = 0; r < R; ++r) {
      ALM_REQUIRE(readings[r] == 1 || readings[r] == 2, ALM_ERR_INVALID,
                  f + ": region " + std::to_string(r) + ": " + std::to_string(readings[r]) +
                      " readings (1 or 2 per region)");
      rstart[static_cast<size_t>(r) + 1] = rstart[static_cast<size_t>(r)] + readings[r];
    }
    ALM_REQUIRE(rstart.back() == N, ALM_ERR_INVALID,
                f + ": the readings sum to " + std::to_string(rstart.back()) + ", not N = " + std::to_string(N));
    const bool want_boxes = lines || kind != ALM_BOX_CROP;
    ALM_REQUIRE(kind == ALM_BOX_QUAD || kind == ALM_BOX_CURVE || (kind == ALM_BOX_CROP && !lines), ALM_ERR_INVALID,
                f + ": kind must be 0 (no boxes), 1 (quad) or 2 (curve); lines need 1 or 2");
    ALM_REQUIRE(!want_boxes || (sizes && geom && n && boxes && centres), ALM_ERR_INVALID,
                f + ": boxes need sizes, geom, n, boxes and centres");
    std::vector<box_core::BoxGeom> g;
    if (want_boxes) {
      g = region_geom(kind, N, sizes, geom, fn);
      for (int i = 0; i < N; ++i) g[static_cast<size_t>(i)].turn = turns[i];
    }
    const MgpSelect sel{R, rstart.data(), turns, turns_out, conf};
    Ctx* c = &h->c;
    c->ensure_ws();
    const size_t sel_bytes = mgp_select_bytes(B, N, R, n_heads, k, want_boxes, lines);
    if (!lines) {
      ALM_REQUIRE(N == B, ALM_ERR_INVALID, f + ": " + std::to_string(N) + " readings for " + std::to_string(B) + " crops");
      ALM_REQUIRE(sel_bytes <= c->ws.cap, ALM_ERR_INVALID,
                  f + ": the readings of " + std::to_string(B) + " crops do not fit in the workspace");
      const MgpBoxes mb{kind, g.empty() ? nullptr : g.data(), n, boxes, centres};
      mgp_forward(c, stage_crops(h, img, B), B, nullptr, nullptr, nullptr, nullptr, ids, probs, k,
                  want_boxes ? &mb : nullptr, nullptr, &sel);
      return;
    }
    ALM_REQUIRE(windows != nullptr, ALM_ERR_INVALID, f + ": lines need windows");
    std::vector<line_core::LineWin> win;
    std::vector<int> wstart(static_cast<size_t>(N) + 1, 0);
    for (int i = 0; i < N; ++i) {
      const box_core::BoxGeom& gi = g[static_cast<size_t>(i)];
      const line_core::Windows w = line_core::line_windows(gi.tw(), gi.th());
      ALM_REQUIRE(windows[i] == w.n, ALM_ERR_INVALID,
                  f + ": reading " + std::to_string(i) + ": " + std::to_string(windows[i]) +
                      " windows, but its turned crop has " + std::to_string(w.n));
      ALM_REQUIRE(wstart[static_cast<size_t>(i)] + w.n <= B, ALM_ERR_INVALID,
                  f + ": the window counts exceed B = " + std::to_string(B));
      for (int j = 0; j < w.n; ++j) win.push_back(line_core::LineWin{i, w.x0[j], w.wn, 0});
      wstart[static_cast<size_t>(i) + 1] = wstart[static_cast<size_t>(i)] + w.n;
    }
    ALM_REQUIRE(wstart.back() == B, ALM_ERR_INVALID,
                f + ": the window counts sum to " + std::to_string(wstart.back()) + ", not B = " + std::to_string(B));
    ALM_REQUIRE(mgp_lines_bytes(B, N) + sel_bytes <= c->ws.cap, ALM_ERR_INVALID,
                f + ": " + std::to_string(B) + " windows do not fit in the workspace");
    const MgpLines ml{kind, N, g.data(), win.data(), wstart.data(), ids, probs, n, boxes, centres};
    mgp_forward(c, stage_crops(h, img, B), B, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, nullptr, &ml,
                &sel);
  });
}

int alm_mgpstr_info(alm_ctx* h, int* dim, int* depth, int* heads, int* n_a3, int* vocab3) {
  return guarded(h, [&] {
    ALM_REQUIRE(h->c.mgp != nullptr, ALM_ERR_STATE, "alm_mgpstr_info before alm_load_weights");
    mgp_info(h->c.mgp, dim, depth, heads, n_a3, vocab3);
  });
}

// ------------------------------------------------------------------------------------------ unit ops
namespace {

// fp32 x [nb][rows][K] as a split-bf16 operand in the workspace, its rows zero-padded to a multiple of 8 elements
Operand split_operand(Ctx* c, const float* x, int rows, int K, int nb) {
  const int Kp = (K + 7) & ~7;
  const size_t n = static_cast<size_t>(nb) * rows * Kp;
  bf16* hi = c->ws.get<bf16>(n);
  bf16* lo = c->ws.get<bf16>(n);
  if (Kp != K)
    for (bf16* p : {hi, lo}) ALM_CHECK_CUDA(cudaMemsetAsync(p, 0, n * 2, c->stream));
  split_rows(c, x, K, static_cast<long>(nb) * rows, K, hi, lo, Kp);
  Operand o;
  o.hi = hi; o.lo = lo; o.rows = rows; o.K = K; o.ld = Kp; o.nb0 = nb; o.bs0 = static_cast<long>(rows) * Kp;
  return o;
}

// A [batch][M][K] times W [w_batch][N][K]^T, both fp32, through the engine's epilogue e
void op_gemm(Ctx* c, const float* A, const float* W, int M, int N, int K, int batch, int w_batch, const Epilogue& e,
             const char* fn) {
  ALM_REQUIRE(K % 4 == 0, ALM_ERR_UNSUPPORTED, std::string(fn) + ": K must be a multiple of 4");
  c->ensure_ws();
  ArenaScope arena_scope(c->ws);
  const Operand a = split_operand(c, A, M, K, batch), b = split_operand(c, W, N, K, w_batch);
  gemm(c, a, b, e);  // its own checks reject the combinations the engine cannot run
  ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
}

// the engine's epilogue for the caller's, once its values and pointers are checked
Epilogue epilogue(const alm_gemm_epilogue& x, const char* fn) {
  ALM_REQUIRE(x.ldo > 0 && x.obs0 >= 0 && x.obs1 >= 0 && x.bias_mode >= BIAS_NONE && x.bias_mode <= BIAS_ROW &&
                  (x.bias != nullptr) == (x.bias_mode != BIAS_NONE) && x.act >= ACT_NONE && x.act <= ACT_RELU &&
                  (!x.out_lo || x.out_hi) && (!x.resid || x.ldr > 0) && x.col_group >= 0,
              ALM_ERR_INVALID, std::string(fn) + " epilogue");
  require_device({x.out_f32, x.out_hi, x.out_lo, x.bias, x.resid, x.resid_map, x.out_map}, 1, fn);
  Epilogue e;
  e.out_f32 = x.out_f32;
  e.out_hi = static_cast<bf16*>(x.out_hi);
  e.out_lo = static_cast<bf16*>(x.out_lo);
  e.ldo = x.ldo; e.obs0 = x.obs0; e.obs1 = x.obs1;
  e.col_group = x.col_group; e.col_group_stride = x.col_group_stride;
  e.bias = x.bias; e.bias_mode = x.bias_mode; e.bias_bs0 = x.bias_bs0;
  e.resid = x.resid; e.ldr = x.resid ? x.ldr : 0; e.rbs0 = x.resid ? x.rbs0 : 0; e.rbs1 = x.resid ? x.rbs1 : 0;
  e.out_map = x.out_map; e.resid_map = x.resid_map;
  e.act = x.act; e.alpha = x.alpha;
  return e;
}

}  // namespace

int alm_op_linear(alm_ctx* h, const float* A, const float* W, const float* bias, float* C, int M, int N, int K, int act,
                  int batch) {
  return guarded(h, [&] {
    ALM_REQUIRE(A && W && C && M > 0 && N > 0 && K > 0 && batch > 0, ALM_ERR_INVALID, "alm_op_linear arguments");
    require_device({A, W, C, bias}, 1, "alm_op_linear");
    Epilogue e;
    e.out_f32 = C; e.ldo = N; e.obs0 = static_cast<long>(M) * N;
    e.bias = bias; e.bias_mode = bias ? BIAS_COL : BIAS_NONE; e.act = act;
    op_gemm(&h->c, A, W, M, N, K, batch, batch, e, "alm_op_linear");
  });
}

int alm_op_gemm(alm_ctx* h, const float* A, const float* W, int M, int N, int K, int batch, int w_batch, float* out_f32,
                void* out_hi, void* out_lo, long ldo, long obs0, const float* bias, int bias_mode, long bias_bs0,
                float alpha, int act, const float* resid, long ldr, long rbs0, const int* resid_map, const int* out_map,
                int col_group, long col_group_stride) {
  return guarded(h, [&] {
    ALM_REQUIRE(A && W && M > 0 && N > 0 && K > 0 && batch > 0 && (w_batch == 1 || w_batch == batch), ALM_ERR_INVALID,
                "alm_op_gemm arguments");
    require_device({A, W}, 1, "alm_op_gemm");
    const alm_gemm_epilogue x{out_f32,   out_hi,   out_lo, ldo, obs0, /*obs1*/ 0, col_group, col_group_stride, bias,
                              bias_mode, bias_bs0, resid,  ldr, rbs0, /*rbs1*/ 0, out_map, resid_map, act, alpha};
    op_gemm(&h->c, A, W, M, N, K, batch, w_batch, epilogue(x, "alm_op_gemm"), "alm_op_gemm");
  });
}

int alm_op_gemm_planes(alm_ctx* h, const alm_gemm_operand* A, const alm_gemm_operand* B, const alm_gemm_epilogue* epi) {
  return guarded(h, [&] {
    ALM_REQUIRE(A && B && epi, ALM_ERR_INVALID, "alm_op_gemm_planes arguments");
    Operand op[2];
    for (int i = 0; i < 2; ++i) {
      const alm_gemm_operand& s = i == 0 ? *A : *B;
      const std::string who = i == 0 ? "alm_op_gemm_planes: A" : "alm_op_gemm_planes: B";
      ALM_REQUIRE(s.hi, ALM_ERR_INVALID, who + " hi plane is null");
      require_device({s.hi, s.lo}, 16, who + " planes");
      ALM_REQUIRE(s.rows > 0 && s.K > 0 && s.ld >= s.K && s.nb0 > 0 && s.nb1 > 0 && s.bs0 >= 0 && s.bs1 >= 0,
                  ALM_ERR_INVALID, who + " extents");
      ALM_REQUIRE(s.ld % 8 == 0 && s.bs0 % 8 == 0 && s.bs1 % 8 == 0, ALM_ERR_INVALID,
                  who + " strides must be multiples of 8 elements");
      ALM_REQUIRE(!s.lo || reinterpret_cast<uintptr_t>(s.lo) > reinterpret_cast<uintptr_t>(s.hi), ALM_ERR_INVALID,
                  who + " lo plane must lie after the hi plane");
      op[i].hi = static_cast<const bf16*>(s.hi);
      op[i].lo = static_cast<const bf16*>(s.lo);
      op[i].rows = s.rows; op[i].K = s.K; op[i].ld = s.ld;
      op[i].nb0 = s.nb0; op[i].nb1 = s.nb1; op[i].bs0 = s.bs0; op[i].bs1 = s.bs1;
    }
    const Epilogue e = epilogue(*epi, "alm_op_gemm_planes");
    Ctx* c = &h->c;
    gemm(c, op[0], op[1], e);  // its own checks reject the batch extents and epilogues the engine cannot run
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  });
}

int alm_op_attention(alm_ctx* h, const float* qkv, float* out, int B, int T, int H) {
  return guarded(h, [&] {
    ALM_REQUIRE(qkv && out && B > 0 && T > 0 && H > 0, ALM_ERR_INVALID, "alm_op_attention arguments");
    require_device({qkv, out}, 1, "alm_op_attention");
    Ctx* c = &h->c;
    c->ensure_ws();
    ArenaScope arena_scope(c->ws);
    const long R = static_cast<long>(B) * T;
    const int D = H * 64;
    bf16* hi = c->ws.get<bf16>(static_cast<size_t>(R) * 3 * D);
    bf16* lo = c->ws.get<bf16>(static_cast<size_t>(R) * 3 * D);
    split_rows(c, qkv, 3 * D, R, 3 * D, hi, lo, 3 * D);
    attention_tc(c, hi, lo, 3L * D, B, T, H, nullptr, nullptr, out, D);
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  });
}

int alm_op_attention_ex(alm_ctx* h, const void* qkv_hi, const void* qkv_lo, long ld, int B, int T, int H, float* out_f32,
                        void* out_hi, void* out_lo, long ldo) {
  return guarded(h, [&] {
    ALM_REQUIRE(qkv_hi && (out_f32 || out_hi) && (!out_lo || out_hi) && B > 0 && T > 0 && H > 0 && ldo >= 64L * H,
                ALM_ERR_INVALID, "alm_op_attention_ex arguments");
    require_device({qkv_hi, qkv_lo, out_f32, out_hi, out_lo}, 16, "alm_op_attention_ex");
    // attention_tc refuses T > 272, ld < 3 H 64, strides that are not multiples of 8 and a missing lo plane at nsplit 3
    Ctx* c = &h->c;
    attention_tc(c, static_cast<const bf16*>(qkv_hi), static_cast<const bf16*>(qkv_lo), ld, B, T, H,
                 static_cast<bf16*>(out_hi), static_cast<bf16*>(out_lo), out_f32, ldo);
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  });
}

int alm_op_row_select(alm_ctx* h, const float* logits, long ld, int rows, int n, int k, int32_t* ids, float* probs) {
  return guarded(h, [&] {
    ALM_REQUIRE(logits && ids && probs, ALM_ERR_INVALID, "alm_op_row_select arguments");
    require_device({logits, ids, probs}, 4, "alm_op_row_select");
    Ctx* c = &h->c;
    mgp_row_select(c, logits, ld, rows, n, k, ids, probs);  // refuses rows or n < 1, n > ld and k outside 0..8
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  });
}

int alm_op_layernorm(alm_ctx* h, const float* x, const float* gamma, const float* beta, float eps, float* y, long rows,
                     int C) {
  return guarded(h, [&] {
    ALM_REQUIRE(x && gamma && beta && y && rows > 0, ALM_ERR_INVALID, "alm_op_layernorm arguments");
    require_device({x, gamma, beta, y}, 1, "alm_op_layernorm");
    gather_ln(&h->c, x, C, nullptr, 1, C, rows, gamma, beta, eps, false, nullptr, 0, y, C, nullptr, nullptr, 0, nullptr,
              nullptr);
    ALM_CHECK_CUDA(cudaStreamSynchronize(h->c.stream));
  });
}

namespace {

// the relative position bias table [169, heads] (device) as the dense [heads, 49, 49] the window kernels read, in the
// workspace (the caller holds the arena scope and synchronizes before it closes)
float* window_bias_dense(Ctx* c, const float* bias_table, int heads) {
  std::vector<float> tab(static_cast<size_t>(169) * heads), dense(static_cast<size_t>(heads) * 2401);
  ALM_CHECK_CUDA(cudaMemcpy(tab.data(), bias_table, tab.size() * 4, cudaMemcpyDeviceToHost));
  for (int hh = 0; hh < heads; ++hh)
    for (int i = 0; i < 49; ++i)
      for (int j = 0; j < 49; ++j)
        dense[static_cast<size_t>(hh) * 2401 + i * 49 + j] =
            tab[static_cast<size_t>((i / 7 - j / 7 + 6) * 13 + (i % 7 - j % 7 + 6)) * heads + hh];
  float* dd = c->ws.get<float>(dense.size());
  ALM_CHECK_CUDA(cudaMemcpyAsync(dd, dense.data(), dense.size() * 4, cudaMemcpyHostToDevice, c->stream));
  return dd;
}

void op_window_attention(alm_ctx* h, const float* qkv, const float* bias_table, float* out_f32, void* out_hi,
                         void* out_lo, int B, int nWh, int nWw, int C, int heads, int shift) {
  ALM_REQUIRE(qkv && bias_table && (out_f32 || out_hi) && (!out_lo || out_hi) && B > 0 && nWh > 0 && nWw > 0 &&
                  heads > 0 && shift >= 0 && shift < 7,
              ALM_ERR_INVALID, "alm_op_window_attention arguments");
  require_device({qkv, bias_table, out_f32}, 16, "alm_op_window_attention");
  require_device({out_hi, out_lo}, 8, "alm_op_window_attention");
  ALM_REQUIRE(C == heads * 32, ALM_ERR_UNSUPPORTED, "alm_op_window_attention: head_dim must be 32");
  {
    Ctx* c = &h->c;
    c->ensure_ws();
    ArenaScope arena_scope(c->ws);
    float* dd = window_bias_dense(c, bias_table, heads);
    window_attention(c, qkv, C, heads, nWh, nWw, B, shift, nWh * 7, nWw * 7, dd, static_cast<bf16*>(out_hi),
                     static_cast<bf16*>(out_lo), out_f32);
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  }
}

}  // namespace

int alm_op_window_attention(alm_ctx* h, const float* qkv, const float* bias_table, float* out, int B, int nWh, int nWw,
                            int C, int heads, int shift) {
  return guarded(h, [&] {
    ALM_REQUIRE(out, ALM_ERR_INVALID, "alm_op_window_attention arguments");
    op_window_attention(h, qkv, bias_table, out, nullptr, nullptr, B, nWh, nWw, C, heads, shift);
  });
}

int alm_op_window_attention_ex(alm_ctx* h, const float* qkv, const float* bias_table, float* out_f32, void* out_hi,
                               void* out_lo, int B, int nWh, int nWw, int C, int heads, int shift) {
  return guarded(h, [&] {
    op_window_attention(h, qkv, bias_table, out_f32, out_hi, out_lo, B, nWh, nWw, C, heads, shift);
  });
}

int alm_op_window_attention_planes(alm_ctx* h, const void* qkv_hi, const void* qkv_lo, const float* bias_table,
                                   float* out_f32, void* out_hi, void* out_lo, int B, int nWh, int nWw, int C, int heads,
                                   int shift) {
  return guarded(h, [&] {
    // both kernels of window_attention_split read the lo plane at every nsplit
    ALM_REQUIRE(qkv_hi && qkv_lo && bias_table && (out_f32 || out_hi) && (!out_lo || out_hi) && B > 0 && nWh > 0 &&
                    nWw > 0 && heads > 0 && shift >= 0 && shift < 7,
                ALM_ERR_INVALID, "alm_op_window_attention_planes arguments");
    require_device({qkv_hi, qkv_lo, bias_table, out_f32}, 16, "alm_op_window_attention_planes");
    require_device({out_hi, out_lo}, 8, "alm_op_window_attention_planes");
    ALM_REQUIRE(C == heads * 32, ALM_ERR_UNSUPPORTED, "alm_op_window_attention_planes: head_dim must be 32");
    Ctx* c = &h->c;
    c->ensure_ws();
    ArenaScope arena_scope(c->ws);
    float* dd = window_bias_dense(c, bias_table, heads);
    window_attention_split(c, static_cast<const bf16*>(qkv_hi), static_cast<const bf16*>(qkv_lo), C, heads, nWh, nWw, B,
                           shift, nWh * 7, nWw * 7, dd, static_cast<bf16*>(out_hi), static_cast<bf16*>(out_lo), out_f32);
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  });
}

namespace {

// alm_op_gather_ln, and with rows_half > 0 its joint form (rows from rows_half on take gamma2 / beta2 / add2)
void op_gather_ln(alm_ctx* h, const float* src, long lds, const int32_t* map, int nsrc, int Cs, long rows,
                  const float* gamma, const float* beta, float eps, int zero_missing, const float* add, long ld_add,
                  float* out_f32, long ldo_f32, void* out_hi, void* out_lo, long ldo_bf, void* out2_hi, void* out2_lo,
                  float* out2_f32, long rows_half, const float* gamma2, const float* beta2, const float* add2) {
  const long C = static_cast<long>(nsrc) * Cs;
  ALM_REQUIRE(src && rows > 0 && nsrc >= 1 && Cs >= 1 && lds >= Cs && (gamma != nullptr) == (beta != nullptr) &&
                  (out_f32 || out_hi || out2_hi || out2_f32) && (!out_lo || out_hi) && (!out2_lo || out2_hi) &&
                  (!add || ((out2_hi || out2_f32) && (ld_add == 0 || ld_add >= C))) &&
                  (!(out_f32 || out2_f32) || ldo_f32 >= C) && (!(out_hi || out2_hi) || ldo_bf >= C) &&
                  (zero_missing == 0 || zero_missing == 1),
              ALM_ERR_INVALID, "alm_op_gather_ln arguments");
  ALM_REQUIRE(lds % 4 == 0 && Cs % 4 == 0 && (!add || ld_add % 4 == 0) && ldo_f32 % 4 == 0 && ldo_bf % 4 == 0,
              ALM_ERR_INVALID, "alm_op_gather_ln: widths and row strides must be multiples of 4");
  require_device({src, gamma, beta, add, out_f32, out2_f32, gamma2, beta2, add2}, 16, "alm_op_gather_ln");
  require_device({map}, 4, "alm_op_gather_ln");
  require_device({out_hi, out_lo, out2_hi, out2_lo}, 8, "alm_op_gather_ln");
  Ctx* c = &h->c;
  gather_ln(c, src, lds, map, nsrc, Cs, rows, gamma, beta, eps, zero_missing != 0, add, ld_add, out_f32, ldo_f32,
            static_cast<bf16*>(out_hi), static_cast<bf16*>(out_lo), ldo_bf, static_cast<bf16*>(out2_hi),
            static_cast<bf16*>(out2_lo), out2_f32, rows_half, gamma2, beta2, add2);
  ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
}

}  // namespace

int alm_op_gather_ln(alm_ctx* h, const float* src, long lds, const int32_t* map, int nsrc, int Cs, long rows,
                     const float* gamma, const float* beta, float eps, int zero_missing, const float* add, long ld_add,
                     float* out_f32, long ldo_f32, void* out_hi, void* out_lo, long ldo_bf, void* out2_hi, void* out2_lo,
                     float* out2_f32) {
  return guarded(h, [&] {
    op_gather_ln(h, src, lds, map, nsrc, Cs, rows, gamma, beta, eps, zero_missing, add, ld_add, out_f32, ldo_f32, out_hi,
                 out_lo, ldo_bf, out2_hi, out2_lo, out2_f32, 0, nullptr, nullptr, nullptr);
  });
}

int alm_op_gather_ln_joint(alm_ctx* h, const float* src, long lds, const int32_t* map, int nsrc, int Cs, long rows,
                           const float* gamma, const float* beta, float eps, int zero_missing, const float* add,
                           long ld_add, float* out_f32, long ldo_f32, void* out_hi, void* out_lo, long ldo_bf,
                           void* out2_hi, void* out2_lo, float* out2_f32, long rows_half, const float* gamma2,
                           const float* beta2, const float* add2) {
  return guarded(h, [&] {
    ALM_REQUIRE(nsrc == 1 && Cs == 512 && rows_half > 0 && rows_half < rows && (gamma2 != nullptr) == (gamma != nullptr) &&
                    (beta2 != nullptr) == (beta != nullptr) && (add2 != nullptr) == (add != nullptr),
                ALM_ERR_INVALID, "alm_op_gather_ln_joint arguments");
    op_gather_ln(h, src, lds, map, nsrc, Cs, rows, gamma, beta, eps, zero_missing, add, ld_add, out_f32, ldo_f32, out_hi,
                 out_lo, ldo_bf, out2_hi, out2_lo, out2_f32, rows_half, gamma2, beta2, add2);
  });
}

int alm_op_swin_map(alm_ctx* h, int kind, int B, int H, int W, int shift, int32_t* map) {
  return guarded(h, [&] {
    ALM_REQUIRE(map && kind >= 0 && kind <= 2 && B > 0 && H > 0 && W > 0 && shift >= 0 && shift < 7 &&
                    (kind == 0 || shift == 0) && static_cast<long>(B) * (H + 6) * (W + 6) < (1L << 31),
                ALM_ERR_INVALID, "alm_op_swin_map arguments");
    require_device({map}, 4, "alm_op_swin_map");
    Ctx* c = &h->c;
    if (kind == 0) window_map(c, map, B, H, W, (H + 6) / 7, (W + 6) / 7, shift);
    else if (kind == 1) merge_map(c, map, B, H, W, (H + 1) / 2, (W + 1) / 2);
    else nearest_map(c, map, B, H, W, (H + 1) / 2, (W + 1) / 2);
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  });
}

int alm_op_patch_im2col(alm_ctx* h, const float* img, int n_canvas, int Hc, int Wc, const int32_t* slots, int B, int H,
                        int W, void* out_hi, void* out_lo) {
  return guarded(h, [&] {
    ALM_REQUIRE(img && out_hi && n_canvas > 0 && B > 0 && H > 0 && W > 0 && H <= Hc && W <= Wc && (slots || B <= n_canvas),
                ALM_ERR_INVALID, "alm_op_patch_im2col arguments");
    require_device({img, slots}, 4, "alm_op_patch_im2col");
    require_device({out_hi, out_lo}, 8, "alm_op_patch_im2col");
    Ctx* c = &h->c;
    if (slots) {  // every image must lie on the canvas
      std::vector<int32_t> s(static_cast<size_t>(B));
      ALM_CHECK_CUDA(cudaMemcpy(s.data(), slots, s.size() * sizeof(int32_t), cudaMemcpyDeviceToHost));
      for (int32_t v : s) ALM_REQUIRE(v >= 0 && v < n_canvas, ALM_ERR_INVALID, "alm_op_patch_im2col: slot out of range");
    }
    im2col_patch4(c, img, B, H, W, (H + 3) / 4, (W + 3) / 4, static_cast<bf16*>(out_hi), static_cast<bf16*>(out_lo), Hc,
                  Wc, slots);
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  });
}

int alm_op_fpn_assemble(alm_ctx* h, const float* p2, const float* p3, const float* p4, const float* p5, int B, int H,
                        int W, void* out_hi, void* out_lo) {
  return guarded(h, [&] {
    ALM_REQUIRE(p2 && p3 && p4 && p5 && out_hi && B > 0 && H > 0 && W > 0, ALM_ERR_INVALID, "alm_op_fpn_assemble arguments");
    require_device({p2, p3, p4, p5}, 16, "alm_op_fpn_assemble");
    require_device({out_hi, out_lo}, 8, "alm_op_fpn_assemble");
    Ctx* c = &h->c;
    int Hs[4], Ws[4];
    stage_grid(H, W, Hs, Ws);
    fpn_assemble(c, p2, p3, p4, p5, B, Hs, Ws, Hs[2], Ws[2], static_cast<bf16*>(out_hi), static_cast<bf16*>(out_lo));
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  });
}

int alm_op_sine_pos(alm_ctx* h, const uint8_t* mask, int B, int H, int W, int hh, int ww, float* pos, uint8_t* kpm) {
  return guarded(h, [&] {
    ALM_REQUIRE(pos && kpm && B > 0 && H > 0 && W > 0 && hh > 0 && ww > 0, ALM_ERR_INVALID, "alm_op_sine_pos arguments");
    require_device({mask, kpm}, 1, "alm_op_sine_pos");
    require_device({pos}, 4, "alm_op_sine_pos");
    Ctx* c = &h->c;
    c->ensure_ws();
    ArenaScope arena_scope(c->ws);
    const std::vector<float> dt = sine_dim_t();
    float* d_dt = c->ws.get<float>(dt.size());
    float* scratch = c->ws.get<float>(static_cast<size_t>(2) * B * hh * ww);
    ALM_CHECK_CUDA(cudaMemcpyAsync(d_dt, dt.data(), dt.size() * sizeof(float), cudaMemcpyHostToDevice, c->stream));
    sine_pos(c, mask, B, H, W, hh, ww, d_dt, pos, kpm, scratch);
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));  // dt goes out of scope
  });
}

int alm_op_softmax_rows(alm_ctx* h, const float* s, long lds, long rows, int n, const uint8_t* kpm, int rows_per_mask,
                        long mask_ld, float* out_f32, void* out_hi, void* out_lo, long ldo) {
  return guarded(h, [&] {
    ALM_REQUIRE(s && rows > 0 && rows < (1L << 31) && n > 0 && lds >= n && ldo >= n && (out_f32 || out_hi) &&
                    (!out_lo || out_hi) && (!kpm || (rows_per_mask > 0 && mask_ld >= n)),
                ALM_ERR_INVALID, "alm_op_softmax_rows arguments");
    require_device({s, out_f32}, 4, "alm_op_softmax_rows");
    require_device({kpm}, 1, "alm_op_softmax_rows");
    require_device({out_hi, out_lo}, 2, "alm_op_softmax_rows");
    Ctx* c = &h->c;
    softmax_rows(c, s, lds, rows, n, kpm, rows_per_mask, mask_ld, out_f32, static_cast<bf16*>(out_hi),
                 static_cast<bf16*>(out_lo), ldo);
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  });
}

namespace {

void op_cross_attention(alm_ctx* h, const float* q, const float* k, const float* v, const uint8_t* kpm, float* out,
                        int nimg_total, int img0, int nimg, int Ncap, int M, int dl, int q_split, int launches,
                        const int* key_len) {
  {
    ALM_REQUIRE(q && k && v && out && nimg_total > 0 && img0 >= 0 && nimg > 0 && img0 + nimg <= nimg_total && Ncap > 0 &&
                    M > 0 && dl >= 0 && dl < 12 && (q_split == 0 || q_split == 1) && launches >= 1,
                ALM_ERR_INVALID, "alm_op_cross_attention arguments");
    ALM_REQUIRE(q_split == 1 || Ncap <= 16, ALM_ERR_INVALID, "alm_op_cross_attention: fp32 queries need Ncap <= 16");
    require_device({q, k, v, out, kpm}, 1, "alm_op_cross_attention");
    Ctx* c = &h->c;
    const int impl = c->xattn_impl;
    ALM_REQUIRE(impl != 1 || Ncap == 1, ALM_ERR_UNSUPPORTED,
                "alm_op_cross_attention: xattn_impl 1 has a fused kernel for one query per image only");
    c->ensure_ws();
    ArenaScope arena_scope(c->ws);
    const DecoderCache kv = decoder_cache(c, k, v, nimg_total, img0, nimg, M, dl, key_len);
    const long slices = static_cast<long>(nimg_total) * 96, koff = kv.off;
    bf16 *kh = kv.kh, *kl = kv.kl, *vh = kv.vh, *vl = kv.vl;
    const long nkv = static_cast<long>(nimg) * M * 512, in_off = static_cast<long>(img0) * M * 512;
    const int Mpad = (M + 7) & ~7;
    bf16 *vth = nullptr, *vtl = nullptr;
    const long voff = (static_cast<long>(img0) * 6144 + dl * 512) * Mpad;
    if (impl == 1) {
      const size_t nvt = static_cast<size_t>(nimg_total) * 6144 * Mpad;
      vth = c->ws.get<bf16>(nvt); vtl = c->ws.get<bf16>(nvt);
      ALM_CHECK_CUDA(cudaMemsetAsync(vth, 0xff, nvt * 2, c->stream));
      ALM_CHECK_CUDA(cudaMemsetAsync(vtl, 0xff, nvt * 2, c->stream));
      op_feature_major_kernel<<<blocks256(nkv), 256, 0, c->stream>>>(v + in_off, M, Mpad, nkv, vth + voff, vtl + voff);
      check_launch("op_feature_major");
    }
    // queries and outputs: fp32 (the skinny form) or split planes (the poly / rec form)
    const long nq = static_cast<long>(nimg) * Ncap * 512;
    bf16 *qh = nullptr, *ql = nullptr, *oh = nullptr, *ol = nullptr;
    if (q_split) {
      qh = c->ws.get<bf16>(nq); ql = c->ws.get<bf16>(nq);
      oh = c->ws.get<bf16>(nq); ol = c->ws.get<bf16>(nq);
      split_rows(c, q, 512, static_cast<long>(nimg) * Ncap, 512, qh, ql, 512);
      ALM_CHECK_CUDA(cudaMemsetAsync(oh, 0xff, nq * 2, c->stream));
      ALM_CHECK_CUDA(cudaMemsetAsync(ol, 0xff, nq * 2, c->stream));
    }
    const float* qf = (q_split && impl != 1) ? nullptr : q;
    float* of = q_split ? nullptr : out;
    const uint8_t* kp = kpm ? kpm + static_cast<long>(img0) * M : nullptr;
    int *d_len = nullptr, *d_off = nullptr;
    if (key_len) {  // keys >= key_len[i] of image i hold NaN in the caches, and the schedule skips their blocks
      std::vector<int> idx(key_len + img0, key_len + img0 + nimg);
      idx.push_back(0);
      for (int i = 0; i < nimg; ++i) idx.push_back(idx.back() + (key_len[img0 + i] + 63) / 64);
      d_len = c->ws.get<int>(idx.size());
      d_off = d_len + nimg;
      ALM_CHECK_CUDA(cudaMemcpyAsync(d_len, idx.data(), idx.size() * sizeof(int), cudaMemcpyHostToDevice, c->stream));
      ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));  // idx goes out of scope
    }
    if (impl == 1) {
      const int ns = cross_attn_q1_splits(c, nimg, M);
      float* partial = c->ws.get<float>(static_cast<size_t>(nimg) * 8 * ns * 66);
      int* counters = c->ws.get<int>(static_cast<size_t>(nimg) * 8);
      fill_i32(c, counters, static_cast<long>(nimg) * 8, 0);
      for (int i = 0; i < launches; ++i)
        cross_attn_q1(c, q, kh + koff, kl + koff, vth + voff, vtl + voff, kp, nimg, M, Mpad, partial, counters, ns, oh, ol, of);
    } else {
      int grid = 0, parts = 0, pairs = 0;
      const int* len = key_len ? key_len + img0 : nullptr;
      if (impl == 2) cross_attn_tma_plan(c, nimg, Ncap, M, &grid, &parts, &pairs, len);
      else cross_attn_mq_plan(c, nimg, Ncap, M, &grid, &parts, &pairs, len);
      const size_t npart = cross_attn_mq_partial_floats(pairs, parts);
      float* partial = c->ws.get<float>(npart);
      int* counters = c->ws.get<int>(pairs);
      ALM_CHECK_CUDA(cudaMemsetAsync(partial, 0xff, npart * 4, c->stream));
      fill_i32(c, counters, pairs, 0);
      for (int i = 0; i < launches; ++i) {
        if (impl == 2)
          cross_attn_tma(c, qh, ql, qf, nimg, Ncap, kh, kl, vh, vl, slices, static_cast<int>(img0 * 96 + dl * 8), kp, M,
                         d_len, d_off, grid, parts, partial, counters, oh, ol, of);
        else
          cross_attn_mq(c, qh, ql, qf, nimg, Ncap, kh + koff, kl + koff, vh + koff, vl + koff, kp, M, d_len, d_off, grid,
                        parts, partial, counters, oh, ol, of);
      }
    }
    if (q_split) {
      op_join_kernel<<<blocks256(nq), 256, 0, c->stream>>>(oh, ol, nq, out);
      check_launch("op_join");
    }
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  }
}

}  // namespace

int alm_op_cross_attention(alm_ctx* h, const float* q, const float* k, const float* v, const uint8_t* kpm, float* out,
                           int nimg_total, int img0, int nimg, int Ncap, int M, int dl, int q_split, int launches) {
  return guarded(h, [&] {
    op_cross_attention(h, q, k, v, kpm, out, nimg_total, img0, nimg, Ncap, M, dl, q_split, launches, nullptr);
  });
}

int alm_op_cross_attention_ex(alm_ctx* h, const float* q, const float* k, const float* v, const uint8_t* kpm, float* out,
                              int nimg_total, int img0, int nimg, int Ncap, int M, int dl, int q_split, int launches,
                              const int* key_len) {
  return guarded(h, [&] {
    ALM_REQUIRE(key_len && img0 >= 0 && nimg > 0 && img0 + nimg <= nimg_total, ALM_ERR_INVALID,
                "alm_op_cross_attention_ex arguments");
    for (int i = img0; i < img0 + nimg; ++i)
      ALM_REQUIRE(key_len[i] >= 1 && key_len[i] <= M, ALM_ERR_INVALID, "alm_op_cross_attention_ex: key_len out of range");
    ALM_REQUIRE(h->c.xattn_impl != 1, ALM_ERR_UNSUPPORTED,
                "alm_op_cross_attention_ex: xattn_impl 1 masks with kpm only and has no per-image key counts");
    op_cross_attention(h, q, k, v, kpm, out, nimg_total, img0, nimg, Ncap, M, dl, q_split, launches, key_len);
  });
}

int alm_op_rec_locations(alm_ctx* h, const float* q, const float* k, const uint8_t* kpm, const int* key_len,
                         const int* mw, float* out, int nimg, int Ncap, int M, int q_split) {
  return guarded(h, [&] {
    ALM_REQUIRE(q && k && mw && out && nimg > 0 && Ncap > 0 && M > 0 && (q_split == 0 || q_split == 1), ALM_ERR_INVALID,
                "alm_op_rec_locations arguments");
    for (int i = 0; i < nimg; ++i)
      ALM_REQUIRE(mw[i] >= 1 && (!key_len || (key_len[i] >= 1 && key_len[i] <= M)), ALM_ERR_INVALID,
                  "alm_op_rec_locations: mw or key_len out of range");
    require_device({q, k, out, kpm}, 1, "alm_op_rec_locations");
    Ctx* c = &h->c;
    c->ensure_ws();
    ArenaScope arena_scope(c->ws);
    const DecoderCache kc = decoder_cache(c, k, nullptr, nimg, 0, nimg, M, 11, key_len);  // the last decoder layer
    // per-image tables: key_len [nimg] (optional), grid widths [nimg]
    std::vector<int> idx(mw, mw + nimg);
    if (key_len) idx.insert(idx.end(), key_len, key_len + nimg);
    int* d_mw = c->ws.get<int>(idx.size());
    const int* d_len = key_len ? d_mw + nimg : nullptr;
    ALM_CHECK_CUDA(cudaMemcpyAsync(d_mw, idx.data(), idx.size() * sizeof(int), cudaMemcpyHostToDevice, c->stream));
    const long nq = static_cast<long>(nimg) * Ncap * 512;
    bf16 *qh = nullptr, *ql = nullptr;
    if (q_split) {
      qh = c->ws.get<bf16>(nq); ql = c->ws.get<bf16>(nq);
      split_rows(c, q, 512, static_cast<long>(nimg) * Ncap, 512, qh, ql, 512);
    }
    int ks = 0, groups = 0;
    size_t pf = 0;
    rec_locate_plan(c, nimg, Ncap, M, key_len, &ks, &pf, &groups);
    float* partial = c->ws.get<float>(pf);
    int* counters = c->ws.get<int>(groups);
    ALM_CHECK_CUDA(cudaMemsetAsync(partial, 0xff, pf * 4, c->stream));
    fill_i32(c, counters, groups, 0);
    rec_locate(c, qh, ql, q_split ? nullptr : q, nimg, Ncap, kc.kh + kc.off, kc.kl + kc.off, kpm, M, d_len, d_mw, ks, partial,
               counters, nullptr, 0, 1, out);
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  });
}

namespace {

// anc: null, or the ancestry of alm_op_self_attention_step_anc
void op_self_attention_step(alm_ctx* h, const float* qkv, float* kc, float* vc, float* out, int S, int t, int Tmax,
                            const int32_t* anc) {
  ALM_REQUIRE(qkv && kc && vc && out && S > 0 && t >= 0 && t < Tmax && Tmax <= 1024, ALM_ERR_INVALID,
              "alm_op_self_attention_step arguments");
  require_device({qkv, kc, vc, out, anc}, 1, "alm_op_self_attention_step");
  Ctx* c = &h->c;
  c->ensure_ws();
  ArenaScope arena_scope(c->ws);
  int* tpos = c->ws.get<int>(1);
  fill_i32(c, tpos, 1, t);
  self_attn_step(c, qkv, qkv + 1024, kc, vc, S, tpos, Tmax, nullptr, nullptr, out, 1536, 1536, anc);
  ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
}

// The decoder loop's token / probability buffers for one step with no prompt: the position counter is gen_index, the
// token lands in column gen_index + 1 and its probability (NaN until written) in column gen_index.  Tmax > 0 adds an
// identity ancestry.
struct StepBuffers {
  int* tokens;
  float* probs;
  int* anc;
  int* tpos;
  int tstride, pstride;
};
StepBuffers step_buffers(Ctx* c, int S, int gen_index, int Tmax) {
  StepBuffers b;
  b.tstride = gen_index + 2;
  b.pstride = gen_index + 1;
  b.tokens = c->ws.get<int>(static_cast<size_t>(S) * b.tstride);
  b.probs = c->ws.get<float>(static_cast<size_t>(S) * b.pstride);
  b.anc = Tmax > 0 ? c->ws.get<int>(static_cast<size_t>(S) * Tmax) : nullptr;
  b.tpos = c->ws.get<int>(1);
  fill_i32(c, b.tokens, static_cast<long>(S) * b.tstride, -1);
  ALM_CHECK_CUDA(cudaMemsetAsync(b.probs, 0xff, static_cast<size_t>(S) * b.pstride * 4, c->stream));
  if (b.anc) anc_identity(c, b.anc, S, Tmax);
  fill_i32(c, b.tpos, 1, gen_index);
  return b;
}

// the step's token and probability of each of the S rows, into the caller's device arrays
void copy_step_out(Ctx* c, const StepBuffers& b, int S, int gen_index, int32_t* token, float* prob) {
  ALM_CHECK_CUDA(cudaMemcpy2DAsync(token, sizeof(int32_t), b.tokens + gen_index + 1, b.tstride * sizeof(int), sizeof(int),
                                   S, cudaMemcpyDeviceToDevice, c->stream));
  ALM_CHECK_CUDA(cudaMemcpy2DAsync(prob, sizeof(float), b.probs + gen_index, b.pstride * sizeof(float), sizeof(float), S,
                                   cudaMemcpyDeviceToDevice, c->stream));
}

}  // namespace

int alm_op_embed_ln(alm_ctx* h, const int32_t* tokens, int tstride, int t, int S, int S_half, const int32_t* tokens2,
                    int tstride2, const float* word_emb, int V, const float* pos_emb, const float* pos_emb2,
                    const float* gamma, const float* beta, float* x, float* qpos, float* qpos2) {
  return guarded(h, [&] {
    const bool joint = S_half != 0;
    ALM_REQUIRE(tokens && word_emb && pos_emb && gamma && beta && x && qpos && S > 0 && V > 0 && t >= 0 && t < 1024 &&
                    tstride > t && S_half >= 0 && S_half < S &&
                    (joint ? tokens2 && pos_emb2 && qpos2 && tstride2 > t : !tokens2 && !pos_emb2 && !qpos2),
                ALM_ERR_INVALID, "alm_op_embed_ln arguments");
    require_device({word_emb, pos_emb, pos_emb2, gamma, beta, x, qpos, qpos2}, 16, "alm_op_embed_ln");
    require_device({tokens, tokens2}, 4, "alm_op_embed_ln");
    Ctx* c = &h->c;
    // the kernel reads column t of each sequence's tokens: every one must be a row of word_emb
    const int n1 = joint ? S_half : S;
    std::vector<int32_t> tok(S);
    ALM_CHECK_CUDA(cudaMemcpy2DAsync(tok.data(), sizeof(int32_t), tokens + t, tstride * sizeof(int32_t), sizeof(int32_t),
                                     n1, cudaMemcpyDeviceToHost, c->stream));
    if (joint)
      ALM_CHECK_CUDA(cudaMemcpy2DAsync(tok.data() + n1, sizeof(int32_t), tokens2 + t, tstride2 * sizeof(int32_t),
                                       sizeof(int32_t), S - n1, cudaMemcpyDeviceToHost, c->stream));
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
    for (int32_t v : tok) ALM_REQUIRE(v >= 0 && v < V, ALM_ERR_INVALID, "alm_op_embed_ln: token outside [0, V)");
    c->ensure_ws();
    ArenaScope arena_scope(c->ws);
    int* tpos = c->ws.get<int>(1);
    fill_i32(c, tpos, 1, t);
    embed_ln(c, tokens, tstride, tpos, S, word_emb, pos_emb, gamma, beta, x, qpos, S_half, tokens2, tstride2, pos_emb2,
             qpos2);
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  });
}

int alm_op_self_attention_step(alm_ctx* h, const float* qkv, float* kc, float* vc, float* out, int S, int t, int Tmax) {
  return guarded(h, [&] { op_self_attention_step(h, qkv, kc, vc, out, S, t, Tmax, nullptr); });
}

int alm_op_self_attention_step_anc(alm_ctx* h, const float* qkv, float* kc, float* vc, float* out, int S, int t, int Tmax,
                                   const int32_t* anc) {
  return guarded(h, [&] {
    ALM_REQUIRE(anc, ALM_ERR_INVALID, "alm_op_self_attention_step_anc: anc is null");
    op_self_attention_step(h, qkv, kc, vc, out, S, t, Tmax, anc);
  });
}

int alm_op_gemv(alm_ctx* h, const float* x, const float* x2, int n_split, const float* W, const float* bias,
                const float* resid, float* out, int M, int N, int K, int act, const float* ln_g, const float* ln_b,
                const float* pos, int pos_split) {
  return guarded(h, [&] {
    ALM_REQUIRE(x && W && out && N > 0 && act >= ACT_NONE && act <= ACT_RELU, ALM_ERR_INVALID, "alm_op_gemv arguments");
    require_device({x, x2, W, bias, resid, out, ln_g, ln_b, pos}, 1, "alm_op_gemv");
    Ctx* c = &h->c;
    gemv_rows(c, x, x2, n_split, K, W, bias, resid, N, out, N, M, N, K, act, ln_g, ln_b, 1e-5f, pos, pos_split);
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  });
}

int alm_op_head_select(alm_ctx* h, const float* logits, int S, int V, int nsoft, int phase, int gen_index,
                       const alm_decode_cfg* cfg, int32_t* token, float* prob, int32_t* finished, int32_t* ntok) {
  return guarded(h, [&] {
    ALM_REQUIRE(logits && cfg && token && prob && S > 0 && V > 0 && nsoft > 0 && nsoft <= V && phase >= 0 && phase <= 2 &&
                    gen_index >= 0 && gen_index < (1 << 20) && (finished == nullptr) == (ntok == nullptr),
                ALM_ERR_INVALID, "alm_op_head_select arguments");
    require_device({logits, token, prob, finished, ntok}, 1, "alm_op_head_select");
    Ctx* c = &h->c;
    c->ensure_ws();
    ArenaScope arena_scope(c->ws);
    const StepBuffers b = step_buffers(c, S, gen_index, 0);  // the pt loop's
    const HeadCfg hc{cfg->num_bins, cfg->pt_eos, cfg->rec_eos, cfg->recog_pad, cfg->vie_categories};
    head_select(c, logits, S, V, nsoft, phase, hc, b.tokens, b.tstride, b.tpos, 0, b.probs, b.pstride, finished, ntok, 1);
    copy_step_out(c, b, S, gen_index, token, prob);
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  });
}

int alm_op_beam_select(alm_ctx* h, const float* logits, int G, int W, int V, int nsoft, int gen_index,
                       const alm_decode_cfg* cfg, float* score, int32_t* len, int32_t* token, int32_t* parent, float* prob) {
  return guarded(h, [&] {
    ALM_REQUIRE(logits && cfg && score && len && token && parent && prob && G > 0 && W >= 1 && W <= ALM_MAX_BEAMS &&
                    V > 0 && nsoft > 0 && nsoft <= V && gen_index >= 0 && gen_index < 1024,
                ALM_ERR_INVALID, "alm_op_beam_select arguments");
    require_device({logits, score, len, token, parent, prob}, 1, "alm_op_beam_select");
    Ctx* c = &h->c;
    c->ensure_ws();
    ArenaScope arena_scope(c->ws);
    // the rec loop's, the parent row in ancestry column gen_index
    const int S = G * W, Tmax = gen_index + 1;
    const StepBuffers b = step_buffers(c, S, gen_index, Tmax);
    const HeadCfg hc{cfg->num_bins, cfg->pt_eos, cfg->rec_eos, cfg->recog_pad, cfg->vie_categories};
    beam_select(c, logits, G, W, V, nsoft, hc, b.tokens, b.tstride, b.tpos, 0, b.probs, b.pstride, score, len, b.anc, Tmax);
    copy_step_out(c, b, S, gen_index, token, prob);
    // the ancestry holds the parent's row; the op reports its slot within the group
    std::vector<int32_t> par(S);
    ALM_CHECK_CUDA(cudaMemcpy2DAsync(par.data(), sizeof(int32_t), b.anc + gen_index, Tmax * sizeof(int), sizeof(int), S,
                                     cudaMemcpyDeviceToHost, c->stream));
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
    for (int r = 0; r < S; ++r) par[r] -= r - r % W;
    ALM_CHECK_CUDA(cudaMemcpy(parent, par.data(), S * sizeof(int32_t), cudaMemcpyHostToDevice));
  });
}

}  // extern "C"
