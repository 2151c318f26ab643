// MGP-STR forward on the GPU: ViT encoder (257 tokens) + three A^3 token learners + char/BPE/WordPiece heads.
// Host-side graph; the arithmetic is the shared wgmma GEMM engine plus the row kernels in kernels.cu.
//
// Reference being replaced (relative to /root/reference/OCR/MGP-STR/): modules/mgp_str.py:64-101,
// modules/token_learner.py:21-32, timm==0.4.12 vision_transformer Block/Attention/Mlp (block LN eps 1e-6,
// scores scaled after q k^T, final norm not applied), demo.py:36-60 (top-1 id + max softmax prob).
#include "mgp.h"

#include <string.h>

#include <algorithm>

#include "block_scan.cuh"
#include "box_core.h"
#include "fuse_core.h"
#include "line_core.h"
#include "omni.h"

#include "ptx.cuh"
#include "topk.cuh"

namespace alm {

struct MgpLin {
  SplitW w;
  float* b = nullptr;
};
struct MgpLN {
  float* g = nullptr;
  float* b = nullptr;
};
struct MgpBlock {
  MgpLN n1, n2;
  MgpLin qkv, proj, fc1, fc2;  // qkv = the packed [3D, D] projection (rows q | k | v), as in the checkpoint
  MgpLin qk, v;                // row views [0, 2D) and [2D, 3D) of qkv for the unfused attention path
};
struct MgpA3 {
  MgpLN token_norm, norm;
  SplitW w0, w1, feat;  // grouped conv [D, D/8], select conv [27, D], grouped feat conv [D, D/8]
  MgpLin head;
  int V = 0, Vpad = 0;
};
struct MgpModel {
  int D = 768, depth = 12, heads = 12;
  MgpLin patch;
  float* cls = nullptr;   // [D]
  float* pos = nullptr;   // [257, D]
  std::vector<MgpBlock> blocks;
  MgpA3 a3[3];
  int n_a3 = 3;  // 3 = MGP-STR (char, bpe, wp); 1 = the char-only CHAR-STR ablation (modules/char_str.py:43-81)
};

void mgp_free(MgpModel* m) { delete m; }
void mgp_info(const MgpModel* m, int* dim, int* depth, int* heads, int* n_a3, int* vocab3) {
  if (dim) *dim = m->D;
  if (depth) *depth = m->depth;
  if (heads) *heads = m->heads;
  if (n_a3) *n_a3 = m->n_a3;
  if (vocab3)
    for (int a = 0; a < 3; ++a) vocab3[a] = a < m->n_a3 ? m->a3[a].V : 0;
}
MgpModel* mgp_share(const MgpModel* owner) { return new MgpModel(*owner); }

namespace {

constexpr int T = 257, TP = 264, NTOK = 27, NPATCH = 256;

MgpLN ld_ln(Ctx* c, const std::map<std::string, HostTensor>& t, const std::string& p, int dim) {
  const HostTensor& g = need(t, p + ".weight");
  const HostTensor& b = need(t, p + ".bias");
  ALM_REQUIRE(static_cast<int>(g.numel()) == dim && static_cast<int>(b.numel()) == dim, ALM_ERR_INVALID,
              "LayerNorm shape mismatch at " + p);
  return MgpLN{upload_f32(c, g.f32.data(), dim), upload_f32(c, b.f32.data(), dim)};
}
MgpLin ld_lin(Ctx* c, const std::map<std::string, HostTensor>& t, const std::string& p, int N, int K, int Kpad = 0) {
  const HostTensor& w = need(t, p + ".weight");
  const HostTensor& b = need(t, p + ".bias");
  ALM_REQUIRE(static_cast<long>(w.numel()) == static_cast<long>(N) * K && static_cast<int>(b.numel()) == N,
              ALM_ERR_INVALID, "Linear shape mismatch at " + p);
  return MgpLin{upload_split(c, w.f32.data(), N, K, Kpad), upload_f32(c, b.f32.data(), N)};
}

__global__ void mgp_patch_maps_kernel(int* out_map, int* resid_map, int B) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= B * NPATCH) return;
  out_map[r] = (r / NPATCH) * T + 1 + r % NPATCH;
  resid_map[r] = 1 + r % NPATCH;
}
// x[b*257 + 0, :] = cls + pos_embed[0]   (mgp_str.py:68-70)
__global__ void mgp_cls_kernel(float* x, const float* cls, const float* pos, int B, int D) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= B * D) return;
  const int b = i / D, d = i % D;
  x[static_cast<long>(b) * T * D + d] = cls[d] + pos[d];
}
// Softmax statistics of one row of n logits, 256 threads: the maximum with its lowest id, and sum_j exp(x_j - max)
// in one fixed reduction order.  The top-1 and the top-k kernels both reduce through here, so the top-k candidate 0
// carries the top-1 kernel's bits.  LIST: every thread also collects its slice's candidates during the max pass.
struct RowSoftmax {
  float max;
  int arg;
  float sum;
};
template <bool LIST>
__device__ __forceinline__ RowSoftmax row_softmax(const float* __restrict__ x, int n, float* sf, int* si, TopkList* l) {
  const int t = threadIdx.x;
  float best = -INFINITY;
  int bi = 0x7fffffff;
  for (int j = t; j < n; j += 256) {
    const float v = x[j];
    if (v > best) { best = v; bi = j; }
    if (LIST) topk_insert(*l, v, j);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; }
  }
  if ((t & 31) == 0) { sf[t >> 5] = best; si[t >> 5] = bi; }
  __syncthreads();
  best = sf[0]; bi = si[0];
#pragma unroll
  for (int i = 1; i < 8; ++i)
    if (sf[i] > best || (sf[i] == best && si[i] < bi)) { best = sf[i]; bi = si[i]; }
  __syncthreads();
  float sum = 0.f;
  for (int j = t; j < n; j += 256) sum += expf(x[j] - best);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((t & 31) == 0) sf[t >> 5] = sum;
  __syncthreads();
  float tot = 0.f;
  for (int i = 0; i < 8; ++i) tot += sf[i];
  return RowSoftmax{best, bi, tot};
}

// per row: argmax id and max softmax probability over n classes (demo.py:36-60)
__global__ void __launch_bounds__(256)
argmax_prob_kernel(const float* __restrict__ logits, long ld, int n, int* __restrict__ ids, float* __restrict__ prob) {
  __shared__ float sf[8];
  __shared__ int si[8];
  const long r = blockIdx.x;
  const RowSoftmax s = row_softmax<false>(logits + r * ld, n, sf, si, nullptr);
  if (threadIdx.x == 0) {
    ids[r] = s.arg;
    prob[r] = 1.0f / s.sum;  // exp(best - best) / sum
  }
}

// per row: the k most likely classes and their softmax probabilities, [row][k] (id -1, prob 0 past the n classes)
__global__ void __launch_bounds__(256)
row_topk_kernel(const float* __restrict__ logits, long ld, int n, int k, int* __restrict__ ids, float* __restrict__ prob) {
  __shared__ float sf[8];
  __shared__ int si[8];
  __shared__ float cv[8 * TOPK_MAX];
  __shared__ int ci[8 * TOPK_MAX];
  const long r = blockIdx.x;
  TopkList l;
  topk_init(l);
  const RowSoftmax s = row_softmax<true>(logits + r * ld, n, sf, si, &l);
  topk_block_merge(l, cv, ci);
  if (threadIdx.x == 0) {
    ids[r * k] = s.arg;  // candidate 0 is argmax_prob_kernel's result (the merged list's head is the same entry)
    prob[r * k] = 1.0f / s.sum;
#pragma unroll
    for (int i = 1; i < TOPK_MAX; ++i) {
      if (i >= k) break;
      const bool none = l.id[i] == 0x7fffffff;
      // ids tied with the maximum get its probability, 1 / sum
      const float e = l.v[i] == s.max ? 1.0f : expf(l.v[i] - s.max);
      ids[r * k + i] = none ? -1 : l.id[i];
      prob[r * k + i] = none ? 0.f : e / s.sum;
    }
  }
}

// per (crop, slot): one A^3 map of this head -> n, box and centre in page coordinates (body in box_core.h).  maps:
// the head's softmaxed selection [B][27][ld], ids: its top-1 ids [B][27][stride] (candidate 0 when stride = k)
__global__ void __launch_bounds__(128)
char_box_kernel(const float* __restrict__ maps, long ld, const int* __restrict__ ids, int stride, int B, int head,
                int kind, const box_core::BoxGeom* __restrict__ geom, int* __restrict__ n, float* __restrict__ boxes,
                float* __restrict__ centres) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long>(B) * box_core::kSlots) return;
  box_core::char_box_slot(i, maps, ld, ids, stride, head, kind, geom, n, boxes, centres);
}

// per (window, slot) of a long line: n, box, centre and line position X of the token (body in line_core.h)
__global__ void __launch_bounds__(128)
line_box_kernel(const float* __restrict__ maps, long ld, const int* __restrict__ ids, int B, int head, int kind,
                const line_core::LineWin* __restrict__ win, const box_core::BoxGeom* __restrict__ geom,
                int* __restrict__ cnt, float* __restrict__ boxes, float* __restrict__ centres, double* __restrict__ X) {
  const long i = static_cast<long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<long>(B) * box_core::kSlots) return;
  line_core::line_box_slot(i, maps, ld, ids, head, kind, win, geom, cnt, boxes, centres, X);
}

// One block per region: thread t < 208 decides slot t (window t / 26, token t % 26 + 1); the kept slots are
// compacted in slot order by a ballot prefix count (no atomics), then every other output position is filled.
__global__ void __launch_bounds__(line_core::kStitchThreads)
line_stitch_kernel(const int* __restrict__ ids, const float* __restrict__ probs, int head,
                   const line_core::LineWin* __restrict__ win, const int* __restrict__ wstart,
                   const int* __restrict__ cnt, const float* __restrict__ boxes, const float* __restrict__ centres,
                   const double* __restrict__ X, int* __restrict__ ids_out, float* __restrict__ probs_out,
                   int* __restrict__ n_out, float* __restrict__ box_out, float* __restrict__ cen_out) {
  __shared__ int warp_kept[line_core::kStitchThreads / 32];
  const int r = blockIdx.x, t = threadIdx.x;
  const int w0 = wstart[r], nw = wstart[r + 1] - w0;
  const bool keep = line_core::stitch_keeps(t, w0, nw, win, cnt, X);
  const block_scan::Rank k = block_scan::ballot_rank<line_core::kStitchThreads>(keep, warp_kept);
  if (keep)
    line_core::stitch_put(r, t, k.pos, w0, ids, probs, boxes, centres, ids_out, probs_out, box_out, cen_out);
  line_core::stitch_fill(r, t, k.total, w0, nw, head, ids, probs, cnt, ids_out, probs_out, box_out, cen_out);
  if (t == 0) n_out[r] = k.total;
}

// Orientation selection (MgpSelect): one output of every head, [n_a3][N][row] 4-byte words on the device, gathered to
// [n_a3][R][row] at the kept readings
struct SelPlane {
  const uint32_t* src;
  uint32_t* dst;
  long row;
};
struct SelArgs {
  const int* ids;       // [n_a3][N][T][stride] top-1 ids (candidate 0 at stride k)
  const float* probs;
  int T, stride, n_a3, N, R;
  const int* rstart;    // [R + 1]
  const int* turns;     // [N]
  SelPlane plane[5];
  int n_plane;
  int* turn_out;        // [R]
  float* conf_out;      // [R]
};
// One block per region: thread i < its readings scores reading i (fuse_core.h's fused confidence over the heads), then
// the block copies the kept reading's row of every plane.
__global__ void __launch_bounds__(128) orient_select_kernel(SelArgs a) {
  __shared__ float conf[2];
  const int r = blockIdx.x, t = threadIdx.x;
  const int r0 = a.rstart[r], nr = a.rstart[r + 1] - r0;
  if (t < nr) conf[t] = fuse_core::reading_conf(a.ids, a.probs, a.T, a.stride, a.n_a3, a.N, r0 + t);
  __syncthreads();
  const int k = fuse_core::pick_reading(conf, a.turns + r0, nr);
  const long s = r0 + k;
  if (t == 0) {
    a.turn_out[r] = a.turns[s];
    a.conf_out[r] = conf[k];
  }
  for (int p = 0; p < a.n_plane; ++p) {
    const SelPlane& q = a.plane[p];
    for (int h = 0; h < a.n_a3; ++h) {
      const uint32_t* src = q.src + (static_cast<long>(h) * a.N + s) * q.row;
      uint32_t* dst = q.dst + (static_cast<long>(h) * a.R + r) * q.row;
      for (long e = t; e < q.row; e += blockDim.x) dst[e] = src[e];
    }
  }
}

struct SB {
  bf16* hi;
  bf16* lo;
};
SB sb(Ctx* c, size_t n) { return SB{c->ws.get<bf16>(n), c->ws.get<bf16>(n)}; }
Operand opnd(const bf16* hi, const bf16* lo, int rows, int K, long ld) {
  Operand o;
  o.hi = hi; o.lo = lo; o.rows = rows; o.K = K; o.ld = ld;
  return o;
}
void lin(Ctx* c, const SB& a, long rows, const MgpLin& l, int act, float* out_f32, SB* out_split, const float* resid) {
  Epilogue e;
  e.out_f32 = out_f32;
  if (out_split) { e.out_hi = out_split->hi; e.out_lo = out_split->lo; }
  e.ldo = l.w.N;
  e.bias = l.b; e.bias_mode = l.b ? BIAS_COL : BIAS_NONE;
  e.act = act;
  e.resid = resid; e.ldr = l.w.N;
  gemm(c, opnd(a.hi, a.lo, static_cast<int>(rows), l.w.K, l.w.K), l.w.op(), e);
}

}  // namespace

void mgp_load(Ctx* c, const std::map<std::string, HostTensor>& tin) {
  // accept 'module.mgp_str.' (DataParallel + Model wrapper, test_final.py:348-356), 'mgp_str.' or bare keys
  std::map<std::string, HostTensor> t;
  for (auto& kv : tin) {
    std::string k = kv.first;
    for (const char* pre : {"module.", "mgp_str."})
      if (k.rfind(pre, 0) == 0) k = k.substr(strlen(pre));
    t.emplace(k, kv.second);
  }
  MgpModel* m = new MgpModel();
  const HostTensor& pe = need(t, "pos_embed");
  ALM_REQUIRE(pe.shape.size() == 3 && pe.shape[1] == T, ALM_ERR_INVALID, "pos_embed must be [1,257,D] (32x128 input, patch 4)");
  m->D = static_cast<int>(pe.shape[2]);
  const int D = m->D;
  // tiny 192 / small 384 / base 768 / large 1024 (mgp_str.py:176-230); every variant has 64-wide heads
  ALM_REQUIRE(D % 64 == 0 && (D % 128 == 0 || D == 192), ALM_ERR_UNSUPPORTED,
              "embed dim must be 192 or a multiple of 128 (tiny=192, small=384, base=768, large=1024)");
  m->heads = D / 64;
  ALM_REQUIRE((D / 8) % 8 == 0, ALM_ERR_UNSUPPORTED, "A^3 group width must be a multiple of 8");
  m->depth = 0;
  while (t.count("blocks." + std::to_string(m->depth) + ".norm1.weight")) ++m->depth;
  ALM_REQUIRE(m->depth > 0, ALM_ERR_INVALID, "no transformer blocks in the state dict");
  m->patch = ld_lin(c, t, "patch_embed.proj", D, 48, 64);
  m->cls = upload_f32(c, need(t, "cls_token").f32.data(), D);
  m->pos = upload_f32(c, pe.f32.data(), static_cast<size_t>(T) * D);
  m->blocks.resize(m->depth);
  for (int b = 0; b < m->depth; ++b) {
    const std::string p = "blocks." + std::to_string(b) + ".";
    MgpBlock& w = m->blocks[b];
    w.n1 = ld_ln(c, t, p + "norm1", D);
    w.n2 = ld_ln(c, t, p + "norm2", D);
    const HostTensor& qw = need(t, p + "attn.qkv.weight");
    const HostTensor& qb = need(t, p + "attn.qkv.bias");
    ALM_REQUIRE(qw.numel() == static_cast<size_t>(3) * D * D && static_cast<int>(qb.numel()) == 3 * D, ALM_ERR_INVALID,
                "qkv shape mismatch at " + p);
    w.qkv.w = upload_split(c, qw.f32.data(), 3 * D, D, 0);
    w.qkv.b = upload_f32(c, qb.f32.data(), 3 * D);
    w.qk = w.qkv; w.qk.w.N = 2 * D;
    w.v = w.qkv; w.v.w.N = D;
    w.v.w.hi += static_cast<size_t>(2) * D * w.qkv.w.ld; w.v.w.lo += static_cast<size_t>(2) * D * w.qkv.w.ld;
    w.v.b += 2 * D;
    w.proj = ld_lin(c, t, p + "attn.proj", D, D);
    w.fc1 = ld_lin(c, t, p + "mlp.fc1", 4 * D, D);
    w.fc2 = ld_lin(c, t, p + "mlp.fc2", D, 4 * D);
  }
  const char* names[3] = {"char", "bpe", "wp"};
  // CHAR-STR (modules/char_str.py:43-81): only the character A^3 module, and its logits come from timm's own
  // classifier `head` (char_str.py:70 calls self.head, not the char_head that reset_classifier creates)
  m->n_a3 = t.count("bpe_tokenLearner.token_norm.weight") ? 3 : 1;
  for (int a = 0; a < m->n_a3; ++a) {
    const std::string p = std::string(names[a]) + "_tokenLearner.";
    MgpA3& w = m->a3[a];
    w.token_norm = ld_ln(c, t, p + "token_norm", D);
    w.norm = ld_ln(c, t, p + "norm", D);
    const HostTensor& w0 = need(t, p + "tokenLearner.0.weight");
    const HostTensor& w1 = need(t, p + "tokenLearner.1.weight");
    const HostTensor& wf = need(t, p + "feat.weight");
    ALM_REQUIRE(w0.numel() == static_cast<size_t>(D) * (D / 8) && wf.numel() == w0.numel() &&
                    w1.numel() == static_cast<size_t>(NTOK) * D, ALM_ERR_INVALID, "A^3 conv shape mismatch at " + p);
    w.w0 = upload_split(c, w0.f32.data(), D, D / 8, 0);
    w.w1 = upload_split(c, w1.f32.data(), NTOK, D, 0);
    w.feat = upload_split(c, wf.f32.data(), D, D / 8, 0);
    const std::string hname = m->n_a3 == 1 ? std::string("head") : std::string(names[a]) + "_head";
    const HostTensor& hw = need(t, hname + ".weight");
    ALM_REQUIRE(hw.shape.size() == 2 && hw.shape[1] == D, ALM_ERR_INVALID, "head shape mismatch");
    w.V = static_cast<int>(hw.shape[0]);
    w.Vpad = (w.V + 7) & ~7;
    w.head = ld_lin(c, t, hname, w.V, D);
  }
  mgp_free(c->mgp);
  c->mgp = m;
}

void mgp_row_select(Ctx* c, const float* logits, long ld, int rows, int n, int k, int32_t* ids, float* prob) {
  ALM_REQUIRE(rows >= 1 && n >= 1 && n <= ld && k >= 0 && k <= TOPK_MAX, ALM_ERR_INVALID, "row selection arguments");
  if (k > 0) {
    row_topk_kernel<<<rows, 256, 0, c->stream>>>(logits, ld, n, k, ids, prob);
    check_launch("row_topk");
  } else {
    argmax_prob_kernel<<<rows, 256, 0, c->stream>>>(logits, ld, n, ids, prob);
    check_launch("argmax_prob");
  }
  count_launch(c);
}

size_t mgp_lines_bytes(int B, int R) {
  const size_t b = static_cast<size_t>(B), r = static_cast<size_t>(R), slots = b * box_core::kSlots;
  const size_t rl = r * line_core::kLineLen, rs = r * line_core::kLineSlots;
  return r * sizeof(box_core::BoxGeom) + b * sizeof(line_core::LineWin) + (r + 1) * sizeof(int) + b * sizeof(int) +
         slots * (10 * sizeof(float) + sizeof(double)) + rl * (sizeof(int) + sizeof(float)) + r * sizeof(int) +
         rs * 10 * sizeof(float) + 12 * 1024;  // 12 allocations, each aligned to 1 KB
}

size_t mgp_select_bytes(int B, int N, int R, int n_a3, int topk, bool boxes, bool lines) {
  const size_t b = static_cast<size_t>(B), n = static_cast<size_t>(N), r = static_cast<size_t>(R);
  const size_t h = static_cast<size_t>(n_a3), per_row = topk > 0 ? static_cast<size_t>(topk) : 1;
  const size_t trow = lines ? line_core::kLineLen : NTOK * per_row;
  const size_t srow = lines ? line_core::kLineSlots : box_core::kSlots;
  // every head's planes, kept until the selection: the stitched lines' planes beyond the first, or the crops' ids /
  // probs and box planes
  size_t kept;
  if (lines)
    kept = (h - 1) * (n * line_core::kLineLen * 8 + n * 4 + n * line_core::kLineSlots * 40);
  else
    kept = 2 * h * b * trow * 4 + (boxes ? h * b * (4 + box_core::kSlots * 40) : 0);
  const size_t select = (r + 1) * 4 + n * 4 + 2 * h * r * trow * 4 + (boxes || lines ? h * r * (4 + srow * 40) : 0) +
                        r * 8;
  return kept + select + 16 * 1024;  // at most 16 allocations, each aligned to 1 KB
}

void mgp_forward(Ctx* c, const float* img, int B, float* attn_out, float* char_logits, float* bpe_logits,
                 float* wp_logits, int32_t* ids_out, float* prob_out, int topk, const MgpBoxes* boxes,
                 const MgpLines* lines, const MgpSelect* orient) {
  MgpModel* m = c->mgp;
  ALM_REQUIRE(m != nullptr, ALM_ERR_STATE, "alm_mgpstr_forward before alm_load_weights");
  ALM_REQUIRE(topk >= 0 && topk <= TOPK_MAX, ALM_ERR_INVALID, "top-k candidates: k must be 1..8");
  ALM_REQUIRE(!lines || topk == 0, ALM_ERR_INVALID, "line stitching follows the top-1 ids");
  ALM_REQUIRE(!orient || !(attn_out || char_logits || bpe_logits || wp_logits), ALM_ERR_INVALID,
              "orientation selection returns no maps or logits");
  c->ensure_ws();
  Arena& ws = c->ws;
  ws.off = 0;
  if (c->omni) c->omni->encoded = false;  // the arena is shared
  const int D = m->D, H = m->heads;
  const long R = static_cast<long>(B) * T;

  float* x = ws.get<float>(R * D);
  // orientation selection: every head's outputs stay in per-head planes (`keep` of them) until the selection
  const int keep = orient ? m->n_a3 : 1;
  const int per_row = topk > 0 ? topk : 1;  // topk > 0: ids / prob hold k candidates per row
  const size_t nsel = static_cast<size_t>(B) * NTOK * per_row;
  int* sel_ids = nullptr;
  float* sel_prob = nullptr;
  if (orient && !lines) {
    sel_ids = ws.get<int>(keep * nsel);
    sel_prob = ws.get<float>(keep * nsel);
  }
  // char boxes: the geometry goes up once; each head's results are copied out before the next head reuses the buffers
  box_core::BoxGeom* bgeom = nullptr;
  int* bn = nullptr;
  float *bbox = nullptr, *bcen = nullptr;
  const long nslot = static_cast<long>(B) * box_core::kSlots;
  if (boxes) {
    bn = ws.get<int>(keep * B);
    bbox = ws.get<float>(keep * nslot * 8);
    bcen = ws.get<float>(keep * nslot * 2);
    if (boxes->geom) {
      bgeom = ws.get<box_core::BoxGeom>(B);
      ALM_CHECK_CUDA(cudaMemcpyAsync(bgeom, boxes->geom, static_cast<size_t>(B) * sizeof(box_core::BoxGeom),
                                     cudaMemcpyHostToDevice, c->stream));
    }
  }
  // long lines: geometry and windows go up once; per head the window boxes land in scratch and only the stitched
  // sequences come back
  struct LineBufs {
    box_core::BoxGeom* geom;
    line_core::LineWin* win;
    int *wstart, *cnt;
    float *wbox, *wcen;
    double* wX;
    int* ids;
    float* probs;
    int* n;
    float *box, *cen;
  } lb{};
  const int LR = lines ? lines->R : 0;
  if (lines) {
    lb.geom = ws.get<box_core::BoxGeom>(LR);
    lb.win = ws.get<line_core::LineWin>(B);
    lb.wstart = ws.get<int>(LR + 1);
    lb.cnt = ws.get<int>(B);
    lb.wbox = ws.get<float>(nslot * 8);
    lb.wcen = ws.get<float>(nslot * 2);
    lb.wX = ws.get<double>(nslot);
    lb.ids = ws.get<int>(keep * static_cast<size_t>(LR) * line_core::kLineLen);
    lb.probs = ws.get<float>(keep * static_cast<size_t>(LR) * line_core::kLineLen);
    lb.n = ws.get<int>(keep * LR);
    lb.box = ws.get<float>(keep * static_cast<size_t>(LR) * line_core::kLineSlots * 8);
    lb.cen = ws.get<float>(keep * static_cast<size_t>(LR) * line_core::kLineSlots * 2);
    ALM_CHECK_CUDA(cudaMemcpyAsync(lb.geom, lines->geom, LR * sizeof(box_core::BoxGeom), cudaMemcpyHostToDevice,
                                   c->stream));
    ALM_CHECK_CUDA(cudaMemcpyAsync(lb.win, lines->win, B * sizeof(line_core::LineWin), cudaMemcpyHostToDevice, c->stream));
    ALM_CHECK_CUDA(cudaMemcpyAsync(lb.wstart, lines->wstart, (LR + 1) * sizeof(int), cudaMemcpyHostToDevice, c->stream));
  }
  // the selection's inputs go up now and its outputs are reserved, so a workspace that is too small fails before the
  // forward runs
  const int N = lines ? LR : B, SR = orient ? orient->R : 0;
  const long trow = lines ? line_core::kLineLen : static_cast<long>(NTOK) * per_row;
  const long srow = lines ? line_core::kLineSlots : box_core::kSlots;
  const bool sel_boxes = lines || boxes;
  struct SelBufs {
    int *rstart, *turns, *ids, *n, *turn;
    float *probs, *box, *cen, *conf;
  } so{};
  if (orient) {
    const size_t hr = static_cast<size_t>(keep) * SR;
    so.rstart = ws.get<int>(SR + 1);
    so.turns = ws.get<int>(N);
    so.ids = ws.get<int>(hr * trow);
    so.probs = ws.get<float>(hr * trow);
    if (sel_boxes) {
      so.n = ws.get<int>(hr);
      so.box = ws.get<float>(hr * srow * 8);
      so.cen = ws.get<float>(hr * srow * 2);
    }
    so.turn = ws.get<int>(SR);
    so.conf = ws.get<float>(SR);
    ALM_CHECK_CUDA(cudaMemcpyAsync(so.rstart, orient->rstart, (SR + 1) * sizeof(int), cudaMemcpyHostToDevice, c->stream));
    ALM_CHECK_CUDA(cudaMemcpyAsync(so.turns, orient->turns, N * sizeof(int), cudaMemcpyHostToDevice, c->stream));
  }
  {  // patch embed + cls + pos (mgp_str.py:66-70)
    const size_t mk = ws.mark();
    SB a = sb(c, static_cast<size_t>(B) * NPATCH * 64);
    int* omap = ws.get<int>(static_cast<size_t>(B) * NPATCH);
    int* rmap = ws.get<int>(static_cast<size_t>(B) * NPATCH);
    im2col_patch4(c, img, B, 32, 128, 8, 32, a.hi, a.lo);
    mgp_patch_maps_kernel<<<(B * NPATCH + 255) / 256, 256, 0, c->stream>>>(omap, rmap, B);
    mgp_cls_kernel<<<(B * D + 255) / 256, 256, 0, c->stream>>>(x, m->cls, m->pos, B, D);
    count_launch(c, 2);
    check_launch("mgp patch maps");
    Epilogue e;
    e.out_f32 = x; e.ldo = D;
    e.bias = m->patch.b; e.bias_mode = BIAS_COL;
    e.resid = m->pos; e.ldr = D; e.out_map = omap; e.resid_map = rmap;
    gemm(c, opnd(a.hi, a.lo, B * NPATCH, 64, 64), m->patch.w.op(), e);
    ws.release(mk);
  }
  const bool fused_attn = c->attn_impl == 0;
  // single-pass bf16 with the fused attention: every consumer (GEMM, attention) reads only the hi planes, so the
  // producers skip computing and writing the lo halves (half of the operand-plane traffic of the ViT)
  struct LoGuard {
    Ctx* c;
    ~LoGuard() { c->lo_unused = false; }
  } lo_guard{c};
  c->lo_unused = (c->nsplit == 1) && fused_attn;
  SB ln = sb(c, R * D);
  SB qk{nullptr, nullptr}, vt{nullptr, nullptr}, P{nullptr, nullptr}, qkv{nullptr, nullptr};
  float* S = nullptr;
  if (fused_attn) {
    qkv = sb(c, R * 3 * D);
  } else {
    qk = sb(c, R * 2 * D);
    vt = sb(c, static_cast<size_t>(B) * D * TP);
    S = ws.get<float>(static_cast<size_t>(B) * H * T * TP);
    P = sb(c, static_cast<size_t>(B) * H * T * TP);
  }
  SB o = sb(c, R * D);
  SB hid = sb(c, R * 4 * D);
  for (int b = 0; b < m->depth; ++b) {
    const MgpBlock& w = m->blocks[b];
    gather_ln(c, x, D, nullptr, 1, D, R, w.n1.g, w.n1.b, 1e-6f, false, nullptr, 0, nullptr, 0, ln.hi, ln.lo, D, nullptr,
              nullptr);
    if (fused_attn) {
      // one packed q|k|v projection, then scores + softmax + P.V in one fused kernel (attn_tc.cu)
      lin(c, ln, R, w.qkv, ACT_NONE, nullptr, &qkv, nullptr);
      attention_tc(c, qkv.hi, qkv.lo, 3L * D, B, T, H, o.hi, o.lo, nullptr, D);
    } else {
    lin(c, ln, R, w.qk, ACT_NONE, nullptr, &qk, nullptr);
    {  // V^T[b, f, t] = Wv ln_b^T + bv  (feature-major: P.V becomes a K-major GEMM)
      Operand bop = opnd(ln.hi, ln.lo, T, D, D);
      bop.nb1 = B; bop.bs1 = static_cast<long>(T) * D;
      Epilogue e;
      e.out_hi = vt.hi; e.out_lo = vt.lo; e.ldo = TP; e.obs1 = static_cast<long>(D) * TP;
      e.bias = w.v.b; e.bias_mode = BIAS_ROW;
      gemm(c, w.v.w.op(), bop, e);
    }
    {  // scores = (q k^T) * 64^-0.5
      Operand q = opnd(qk.hi, qk.lo, T, 64, 2 * D);
      q.nb0 = H; q.bs0 = 64; q.nb1 = B; q.bs1 = static_cast<long>(T) * 2 * D;
      Operand k = q;
      k.hi = qk.hi + D; k.lo = qk.lo + D;
      Epilogue e;
      e.out_f32 = S; e.ldo = TP; e.obs0 = static_cast<long>(T) * TP; e.obs1 = static_cast<long>(H) * T * TP;
      e.alpha = 0.125f;
      gemm(c, q, k, e);
    }
    softmax_rows(c, S, TP, static_cast<long>(B) * H * T, T, nullptr, 1, 0, nullptr, P.hi, P.lo, TP);
    {
      Operand p = opnd(P.hi, P.lo, T, T, TP);
      p.nb0 = H; p.bs0 = static_cast<long>(T) * TP; p.nb1 = B; p.bs1 = static_cast<long>(H) * T * TP;
      Operand v = opnd(vt.hi, vt.lo, 64, T, TP);
      v.nb0 = H; v.bs0 = static_cast<long>(64) * TP; v.nb1 = B; v.bs1 = static_cast<long>(D) * TP;
      Epilogue e;
      e.out_hi = o.hi; e.out_lo = o.lo; e.ldo = D; e.obs0 = 64; e.obs1 = static_cast<long>(T) * D;
      gemm(c, p, v, e);
    }
    }  // unfused attention
    lin(c, o, R, w.proj, ACT_NONE, x, nullptr, x);
    gather_ln(c, x, D, nullptr, 1, D, R, w.n2.g, w.n2.b, 1e-6f, false, nullptr, 0, nullptr, 0, ln.hi, ln.lo, D, nullptr,
              nullptr);
    lin(c, ln, R, w.fc1, ACT_GELU, nullptr, &hid, nullptr);
    lin(c, hid, R, w.fc2, ACT_NONE, x, nullptr, x);
  }
  // ---- three A^3 modules + heads (token_learner.py:21-32, mgp_str.py:79-92)
  const size_t a3_mark = ws.mark();
  float* logit_dst[3] = {char_logits, bpe_logits, wp_logits};
  const int G = 8, Dg = D / 8;
  for (int a = 0; a < m->n_a3; ++a) {
    ws.release(a3_mark);
    const MgpA3& w = m->a3[a];
    SB tn = sb(c, R * D);
    SB s0 = sb(c, R * D);
    float* sel = ws.get<float>(static_cast<size_t>(B) * NTOK * TP);
    float* attn = ws.get<float>(static_cast<size_t>(B) * NTOK * TP);
    SB Pa = sb(c, static_cast<size_t>(B) * NTOK * TP);
    SB ft = sb(c, static_cast<size_t>(B) * D * TP);
    float* xa = ws.get<float>(static_cast<size_t>(B) * NTOK * D);
    SB xn = sb(c, static_cast<size_t>(B) * NTOK * D);
    float* logits = ws.get<float>(static_cast<size_t>(B) * NTOK * w.Vpad);
    int* ids = sel_ids ? sel_ids + a * nsel : ws.get<int>(nsel);
    float* prob = sel_prob ? sel_prob + a * nsel : ws.get<float>(nsel);
    gather_ln(c, x, D, nullptr, 1, D, R, w.token_norm.g, w.token_norm.b, 1e-5f, false, nullptr, 0, nullptr, 0, tn.hi,
              tn.lo, D, nullptr, nullptr);
    {  // grouped 1x1 conv (8 groups): per group a [R, Dg] x [Dg, Dg]^T GEMM
      Operand aop = opnd(tn.hi, tn.lo, static_cast<int>(R), Dg, D);
      aop.nb0 = G; aop.bs0 = Dg;
      Operand wop = opnd(w.w0.hi, w.w0.lo, Dg, Dg, Dg);
      wop.nb0 = G; wop.bs0 = static_cast<long>(Dg) * Dg;
      Epilogue e;
      e.out_hi = s0.hi; e.out_lo = s0.lo; e.ldo = D; e.obs0 = Dg;
      gemm(c, aop, wop, e);
    }
    {  // selected^T[b, s, t] = W1 s0_b^T
      Operand bop = opnd(s0.hi, s0.lo, T, D, D);
      bop.nb1 = B; bop.bs1 = static_cast<long>(T) * D;
      Epilogue e;
      e.out_f32 = sel; e.ldo = TP; e.obs1 = static_cast<long>(NTOK) * TP;
      gemm(c, w.w1.op(), bop, e);
    }
    softmax_rows(c, sel, TP, static_cast<long>(B) * NTOK, T, nullptr, 1, 0, attn, Pa.hi, Pa.lo, TP);
    {  // feat^T[b, g*Dg + f, t] = Wf_g tn_b[:, g]^T
      Operand aop = opnd(w.feat.hi, w.feat.lo, Dg, Dg, Dg);
      aop.nb0 = G; aop.bs0 = static_cast<long>(Dg) * Dg;
      Operand bop = opnd(tn.hi, tn.lo, T, Dg, D);
      bop.nb0 = G; bop.bs0 = Dg; bop.nb1 = B; bop.bs1 = static_cast<long>(T) * D;
      Epilogue e;
      e.out_hi = ft.hi; e.out_lo = ft.lo; e.ldo = TP; e.obs0 = static_cast<long>(Dg) * TP; e.obs1 = static_cast<long>(D) * TP;
      gemm(c, aop, bop, e);
    }
    {  // x_a[b] = selected[b] (27 x 257) . feat[b] (257 x D)
      Operand aop = opnd(Pa.hi, Pa.lo, NTOK, T, TP);
      aop.nb1 = B; aop.bs1 = static_cast<long>(NTOK) * TP;
      Operand bop = opnd(ft.hi, ft.lo, D, T, TP);
      bop.nb1 = B; bop.bs1 = static_cast<long>(D) * TP;
      Epilogue e;
      e.out_f32 = xa; e.ldo = D; e.obs1 = static_cast<long>(NTOK) * D;
      gemm(c, aop, bop, e);
    }
    gather_ln(c, xa, D, nullptr, 1, D, static_cast<long>(B) * NTOK, w.norm.g, w.norm.b, 1e-5f, false, nullptr, 0, nullptr,
              0, xn.hi, xn.lo, D, nullptr, nullptr);
    {
      Epilogue e;
      e.out_f32 = logits; e.ldo = w.Vpad;
      e.bias = w.head.b; e.bias_mode = BIAS_COL;
      gemm(c, opnd(xn.hi, xn.lo, B * NTOK, D, D), w.head.w.op(), e);
    }
    mgp_row_select(c, logits, w.Vpad, B * NTOK, w.V, topk, ids, prob);
    const int ka = orient ? a : 0;  // this head's plane of the kept outputs
    if (boxes) {  // the maps and ids of this head are still in the workspace
      char_box_kernel<<<static_cast<unsigned>((nslot + 127) / 128), 128, 0, c->stream>>>(
          attn, TP, ids, per_row, B, a, boxes->kind, bgeom, bn + ka * B, bbox + ka * nslot * 8, bcen + ka * nslot * 2);
      count_launch(c);
      check_launch("char_box");
    }
    if (boxes && !orient) {
      ALM_CHECK_CUDA(cudaMemcpyAsync(boxes->n + static_cast<size_t>(a) * B, bn, B * sizeof(int), cudaMemcpyDeviceToHost,
                                     c->stream));
      ALM_CHECK_CUDA(cudaMemcpyAsync(boxes->boxes + static_cast<size_t>(a) * nslot * 8, bbox, nslot * 8 * sizeof(float),
                                     cudaMemcpyDeviceToHost, c->stream));
      ALM_CHECK_CUDA(cudaMemcpyAsync(boxes->centres + static_cast<size_t>(a) * nslot * 2, bcen,
                                     nslot * 2 * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    }
    const size_t rl = static_cast<size_t>(LR) * line_core::kLineLen, rs = static_cast<size_t>(LR) * line_core::kLineSlots;
    if (lines) {  // window boxes, then the stitch, while this head's maps, ids and probabilities are in the workspace
      line_box_kernel<<<static_cast<unsigned>((nslot + 127) / 128), 128, 0, c->stream>>>(
          attn, TP, ids, B, a, lines->kind, lb.win, lb.geom, lb.cnt, lb.wbox, lb.wcen, lb.wX);
      count_launch(c);
      check_launch("line_box");
      line_stitch_kernel<<<LR, line_core::kStitchThreads, 0, c->stream>>>(
          ids, prob, a, lb.win, lb.wstart, lb.cnt, lb.wbox, lb.wcen, lb.wX, lb.ids + ka * rl, lb.probs + ka * rl,
          lb.n + ka * LR, lb.box + ka * rs * 8, lb.cen + ka * rs * 2);
      count_launch(c);
      check_launch("line_stitch");
    }
    if (lines && !orient) {
      ALM_CHECK_CUDA(cudaMemcpyAsync(lines->ids + a * rl, lb.ids, rl * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
      ALM_CHECK_CUDA(cudaMemcpyAsync(lines->probs + a * rl, lb.probs, rl * sizeof(float), cudaMemcpyDeviceToHost,
                                     c->stream));
      ALM_CHECK_CUDA(cudaMemcpyAsync(lines->n + static_cast<size_t>(a) * LR, lb.n, LR * sizeof(int),
                                     cudaMemcpyDeviceToHost, c->stream));
      ALM_CHECK_CUDA(cudaMemcpyAsync(lines->boxes + a * rs * 8, lb.box, rs * 8 * sizeof(float), cudaMemcpyDeviceToHost,
                                     c->stream));
      ALM_CHECK_CUDA(cudaMemcpyAsync(lines->centres + a * rs * 2, lb.cen, rs * 2 * sizeof(float),
                                     cudaMemcpyDeviceToHost, c->stream));
    }
    const size_t rows = static_cast<size_t>(B) * NTOK;
    if (attn_out)
      ALM_CHECK_CUDA(cudaMemcpy2DAsync(attn_out + static_cast<size_t>(a) * rows * T, T * sizeof(float), attn,
                                       TP * sizeof(float), T * sizeof(float), rows, cudaMemcpyDeviceToHost, c->stream));
    if (logit_dst[a])
      ALM_CHECK_CUDA(cudaMemcpy2DAsync(logit_dst[a], w.V * sizeof(float), logits, w.Vpad * sizeof(float),
                                       w.V * sizeof(float), rows, cudaMemcpyDeviceToHost, c->stream));
    if (ids_out && !orient)
      ALM_CHECK_CUDA(cudaMemcpyAsync(ids_out + a * nsel, ids, nsel * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    if (prob_out && !orient)
      ALM_CHECK_CUDA(cudaMemcpyAsync(prob_out + a * nsel, prob, nsel * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
    ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));  // buffers are reused by the next head
  }
  if (!orient) return;
  // one reading per region: score, pick and gather on the device; only the R kept rows cross PCIe
  SelArgs sa{};
  sa.ids = lines ? lb.ids : sel_ids;
  sa.probs = lines ? lb.probs : sel_prob;
  sa.T = lines ? line_core::kLineLen : NTOK;
  sa.stride = lines ? 1 : per_row;
  sa.n_a3 = m->n_a3; sa.N = N; sa.R = SR;
  sa.rstart = so.rstart; sa.turns = so.turns;
  auto plane = [&](const void* src, void* dst, long row) {
    sa.plane[sa.n_plane++] = SelPlane{static_cast<const uint32_t*>(src), static_cast<uint32_t*>(dst), row};
  };
  plane(sa.ids, so.ids, trow);
  plane(sa.probs, so.probs, trow);
  if (sel_boxes) {
    plane(lines ? lb.n : bn, so.n, 1);
    plane(lines ? lb.box : bbox, so.box, srow * 8);
    plane(lines ? lb.cen : bcen, so.cen, srow * 2);
  }
  sa.turn_out = so.turn; sa.conf_out = so.conf;
  orient_select_kernel<<<SR, 128, 0, c->stream>>>(sa);
  count_launch(c);
  check_launch("orient_select");
  const size_t hr = static_cast<size_t>(m->n_a3) * SR;
  auto down = [&](void* dst, const void* src, size_t bytes) {
    if (dst) ALM_CHECK_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, c->stream));
  };
  down(lines ? lines->ids : ids_out, so.ids, hr * trow * sizeof(int));
  down(lines ? lines->probs : prob_out, so.probs, hr * trow * sizeof(float));
  if (sel_boxes) {
    down(lines ? lines->n : boxes->n, so.n, hr * sizeof(int));
    down(lines ? lines->boxes : boxes->boxes, so.box, hr * srow * 8 * sizeof(float));
    down(lines ? lines->centres : boxes->centres, so.cen, hr * srow * 2 * sizeof(float));
  }
  down(orient->turn_out, so.turn, SR * sizeof(int));
  down(orient->conf_out, so.conf, SR * sizeof(float));
  ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
}

}  // namespace alm
