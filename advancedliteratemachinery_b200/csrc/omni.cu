// OmniParser forward on the GPU: Swin-B encoder -> FPN -> input_proj -> three KV-cached point-conditioned
// decoders.  This file is the host-side graph (sequence of kernel launches on the context stream); the
// arithmetic lives in gemm.cu / kernels.cu / omni_kernels.cu.
//
// Reference being replaced (relative to /root/reference/OCR/OmniParser/):
//   model/omniparser.py:19-32, model/backbone/swin_transformer.py:597-625, model/fpn.py:21-45,
//   model/backbone/position_embedding.py:24-44, model/transformer.py:74-141,219-286.
#include <math.h>

#include <algorithm>
#include <cmath>
#include <optional>
#include <unordered_map>
#include <string>

#include "dense_core.h"
#include "omni.h"
#include "pre.h"

namespace alm {

SplitW upload_split(Ctx* c, const float* w, int N, int K, int Kpad);

namespace {

const int kDepths[4] = {2, 2, 18, 2};
const int kHeads[4] = {4, 8, 16, 32};

LNW load_ln(Ctx* c, const std::map<std::string, HostTensor>& t, const std::string& p, int dim) {
  const HostTensor& g = need(t, p + ".weight");
  const HostTensor& b = need(t, p + ".bias");
  ALM_REQUIRE(static_cast<int>(g.numel()) == dim && static_cast<int>(b.numel()) == dim, ALM_ERR_INVALID,
              "LayerNorm shape mismatch at " + p);
  LNW l;
  l.g = upload_f32(c, g.f32.data(), dim);
  l.b = upload_f32(c, b.f32.data(), dim);
  return l;
}

Lin load_lin(Ctx* c, const std::map<std::string, HostTensor>& t, const std::string& p, int N, int K, bool bias = true,
             int Kpad = 0, bool keep_f32 = false) {
  const HostTensor& w = need(t, p + ".weight");
  ALM_REQUIRE(static_cast<long>(w.numel()) == static_cast<long>(N) * K, ALM_ERR_INVALID,
              "Linear weight shape mismatch at " + p);
  Lin l;
  l.w = upload_split(c, w.f32.data(), N, K, Kpad);
  if (keep_f32) l.wf = upload_f32(c, w.f32.data(), w.numel());
  if (bias) {
    const HostTensor& b = need(t, p + ".bias");
    ALM_REQUIRE(static_cast<int>(b.numel()) == N, ALM_ERR_INVALID, "Linear bias shape mismatch at " + p);
    l.b = upload_f32(c, b.f32.data(), N);
  }
  return l;
}

// Swin qkv projection with the attention scale folded into the q rows (swin_transformer.py:130 multiplies q by
// head_dim^-0.5 right after the projection): the GEMM epilogue then emits the operand planes of q*scale directly
Lin load_qkv_qscaled(Ctx* c, const std::map<std::string, HostTensor>& t, const std::string& p, int C) {
  const HostTensor& w = need(t, p + ".weight");
  const HostTensor& b = need(t, p + ".bias");
  ALM_REQUIRE(static_cast<long>(w.numel()) == 3L * C * C && static_cast<long>(b.numel()) == 3L * C, ALM_ERR_INVALID,
              "qkv shape mismatch at " + p);
  std::vector<float> ws(w.f32), bs(b.f32);
  for (size_t i = 0; i < static_cast<size_t>(C) * C; ++i) ws[i] *= WATTN_QSCALE;
  for (int i = 0; i < C; ++i) bs[i] *= WATTN_QSCALE;
  Lin l;
  l.w = upload_split(c, ws.data(), 3 * C, C, 0);
  l.b = upload_f32(c, bs.data(), bs.size());
  return l;
}

// rows [r0, r0+n) of a packed in_proj weight/bias
Lin load_inproj_rows(Ctx* c, const std::map<std::string, HostTensor>& t, const std::string& p, int r0, int n) {
  const HostTensor& w = need(t, p + ".in_proj_weight");
  const HostTensor& b = need(t, p + ".in_proj_bias");
  ALM_REQUIRE(w.numel() == size_t(1536) * 512 && b.numel() == 1536, ALM_ERR_INVALID, "in_proj shape mismatch at " + p);
  Lin l;
  l.w = upload_split(c, w.f32.data() + static_cast<size_t>(r0) * 512, n, 512, 0);
  l.wf = upload_f32(c, w.f32.data() + static_cast<size_t>(r0) * 512, static_cast<size_t>(n) * 512);
  l.b = upload_f32(c, b.f32.data() + r0, n);
  return l;
}

// The same linear of the polygon and the recognition decoder (p[0], p[1]) as one [2N, K] slab, bias [2N] and fp32
// copy likewise: out[1] is out[0] + N rows, so one GEMM with a batch dimension of 2 (B stride N * K) runs both.
// Plain (unpaired) weights of the point decoder keep their own slabs.  rows [r0, r0 + N) of a packed in_proj when
// inproj, else the whole `.weight` / `.bias`.
void load_lin_pair(Ctx* c, const std::map<std::string, HostTensor>& t, const std::string p[2], int N, int K, bool inproj,
                   int r0, Lin out[2]) {
  std::vector<float> w(static_cast<size_t>(2) * N * K), b(static_cast<size_t>(2) * N);
  for (int i = 0; i < 2; ++i) {
    const HostTensor& hw = need(t, p[i] + (inproj ? ".in_proj_weight" : ".weight"));
    const HostTensor& hb = need(t, p[i] + (inproj ? ".in_proj_bias" : ".bias"));
    ALM_REQUIRE(inproj ? (hw.numel() == size_t(1536) * 512 && hb.numel() == 1536)
                       : (static_cast<long>(hw.numel()) == static_cast<long>(N) * K && static_cast<int>(hb.numel()) == N),
                ALM_ERR_INVALID, "Linear shape mismatch at " + p[i]);
    std::copy(hw.f32.begin() + static_cast<size_t>(r0) * K, hw.f32.begin() + static_cast<size_t>(r0 + N) * K,
              w.begin() + static_cast<size_t>(i) * N * K);
    std::copy(hb.f32.begin() + r0, hb.f32.begin() + r0 + N, b.begin() + static_cast<size_t>(i) * N);
  }
  const SplitW sw = upload_split(c, w.data(), 2 * N, K, 0);
  float* wf = upload_f32(c, w.data(), w.size());
  float* bf = upload_f32(c, b.data(), b.size());
  for (int i = 0; i < 2; ++i) {
    const size_t off = static_cast<size_t>(i) * N * sw.ld;
    out[i].w = sw;
    out[i].w.N = N;
    out[i].w.hi = sw.hi + off;
    out[i].w.lo = sw.lo + off;
    out[i].wf = wf + static_cast<size_t>(i) * N * K;
    out[i].b = bf + static_cast<size_t>(i) * N;
  }
}

Operand act_op(const bf16* hi, const bf16* lo, long rows, int K, long ld) {
  Operand o;
  o.hi = hi; o.lo = lo; o.rows = static_cast<int>(rows); o.K = K; o.ld = ld;
  return o;
}

struct SplitBuf {
  bf16* hi = nullptr;
  bf16* lo = nullptr;
};
SplitBuf alloc_split(Ctx* c, size_t n) {
  SplitBuf s;
  s.hi = c->ws.get<bf16>(n);
  s.lo = c->ws.get<bf16>(n);
  return s;
}

void linear(Ctx* c, const SplitBuf& a, long rows, const Lin& l, int act, float* out_f32, SplitBuf* out_split,
            const float* resid = nullptr, const int* out_map = nullptr, const int* resid_map = nullptr, long ldr = 0) {
  Epilogue e;
  e.out_f32 = out_f32;
  if (out_split) { e.out_hi = out_split->hi; e.out_lo = out_split->lo; }
  e.ldo = l.w.N;
  e.bias = l.b;
  e.bias_mode = l.b ? BIAS_COL : BIAS_NONE;
  e.act = act;
  e.resid = resid;
  e.ldr = ldr ? ldr : l.w.N;
  e.out_map = out_map;
  e.resid_map = resid_map;
  gemm(c, act_op(a.hi, a.lo, rows, l.w.K, l.w.K), l.w.op(), e);
}

// The same linear of the polygon and the recognition decoder over the two halves of a joint decoder pass: rows [0, S)
// of `a` / the outputs take l0, rows [S, 2S) take l1 (loaded as one slab, load_lin_pair).  One GEMM with a batch
// dimension of 2: each row's arithmetic is that of linear() with its own decoder's weights.
void linear2(Ctx* c, const SplitBuf& a, long S, const Lin& l0, const Lin& l1, int act, float* out_f32, SplitBuf* out_split,
             const float* resid = nullptr) {
  const int N = l0.w.N, K = l0.w.K;
  Operand A = act_op(a.hi, a.lo, S, K, K);
  A.nb0 = 2; A.bs0 = S * K;
  Operand W = l0.w.op();
  W.nb0 = 2; W.bs0 = l1.w.hi - l0.w.hi;
  ALM_REQUIRE(l1.w.N == N && l1.w.K == K && l1.w.lo - l0.w.lo == W.bs0 && l1.b - l0.b == N, ALM_ERR_STATE,
              "joint decoder linear: the two decoders' weights are not one slab");
  Epilogue e;
  e.out_f32 = out_f32;
  if (out_split) { e.out_hi = out_split->hi; e.out_lo = out_split->lo; }
  e.ldo = N; e.obs0 = S * N;
  e.bias = l0.b; e.bias_mode = BIAS_COL; e.bias_bs0 = N;
  e.act = act;
  e.resid = resid; e.ldr = N; e.rbs0 = resid ? S * N : 0;
  gemm(c, A, W, e);
}

}  // namespace

// ================================================================================================ load
void omni_load(Ctx* c, int kind, const std::map<std::string, HostTensor>& t) {
  OmniModel* m = new OmniModel();
  const std::string bb = "backbone.0.";
  m->patch = load_lin(c, t, bb + "patch_embed.proj", 128, 48, true, 64);
  m->patch_norm = load_ln(c, t, bb + "patch_embed.norm", 128);
  // relative_position_index [49,49] (swin_transformer.py:98-109): recomputed, then cross-checked if present
  std::vector<int> rel_index(49 * 49);
  for (int i = 0; i < 49; ++i)
    for (int j = 0; j < 49; ++j)
      rel_index[i * 49 + j] = (i / 7 - j / 7 + 6) * 13 + (i % 7 - j % 7 + 6);
  for (int s = 0; s < 4; ++s) {
    const int C = 128 << s, heads = kHeads[s];
    m->stage[s].blocks.resize(kDepths[s]);
    for (int b = 0; b < kDepths[s]; ++b) {
      const std::string p = bb + "layers." + std::to_string(s) + ".blocks." + std::to_string(b) + ".";
      SwinBlockW& w = m->stage[s].blocks[b];
      w.n1 = load_ln(c, t, p + "norm1", C);
      w.n2 = load_ln(c, t, p + "norm2", C);
      w.qkv = load_qkv_qscaled(c, t, p + "attn.qkv", C);
      w.proj = load_lin(c, t, p + "attn.proj", C, C);
      w.fc1 = load_lin(c, t, p + "mlp.fc1", 4 * C, C);
      w.fc2 = load_lin(c, t, p + "mlp.fc2", C, 4 * C);
      const HostTensor& tab = need(t, p + "attn.relative_position_bias_table");
      ALM_REQUIRE(static_cast<int>(tab.numel()) == 169 * heads, ALM_ERR_INVALID, "bias table shape mismatch at " + p);
      auto it = t.find(p + "attn.relative_position_index");
      if (it != t.end() && !it->second.placeholder) {
        ALM_REQUIRE(it->second.numel() == 49 * 49, ALM_ERR_INVALID, "relative_position_index shape at " + p);
        for (int i = 0; i < 49 * 49; ++i)
          ALM_REQUIRE(static_cast<int>(it->second.f32[i]) == rel_index[i], ALM_ERR_INVALID,
                      "relative_position_index differs from the Swin definition at " + p);
      }
      std::vector<float> dense(static_cast<size_t>(heads) * 49 * 49);
      for (int h = 0; h < heads; ++h)
        for (int i = 0; i < 49 * 49; ++i) dense[static_cast<size_t>(h) * 2401 + i] = tab.f32[rel_index[i] * heads + h];
      w.bias_dense = upload_f32(c, dense.data(), dense.size());
    }
    m->stage[s].out_norm = load_ln(c, t, bb + "norm" + std::to_string(s), C);
    if (s < 3) {
      const std::string p = bb + "layers." + std::to_string(s) + ".downsample.";
      m->stage[s].merge_norm = load_ln(c, t, p + "norm", 4 * C);
      m->stage[s].merge_red = load_lin(c, t, p + "reduction", 2 * C, 4 * C, false).w;
    }
  }
  const int fpn_in[4] = {1024, 512, 256, 128};
  for (int i = 0; i < 4; ++i) m->fpn[i] = load_lin(c, t, "fpn.fpn_in." + std::to_string(i), 256, fpn_in[i], false).w;
  m->inproj = load_lin(c, t, "input_proj", 512, 1024);
  {
    const std::vector<float> dt = sine_dim_t();
    m->dim_t = upload_f32(c, dt.data(), dt.size());
  }
  // ---- decoder
  const std::string tr = "transformer.";
  const HostTensor& we = need(t, tr + "embedding.word_embeddings.weight");
  ALM_REQUIRE(we.shape.size() == 2 && we.shape[1] == 512, ALM_ERR_INVALID, "word_embeddings shape");
  m->V = static_cast<int>(we.shape[0]);
  m->vie = m->V - 1104;
  ALM_REQUIRE(m->vie >= 0, ALM_ERR_INVALID, "vocabulary smaller than the text-spotting layout (1104)");
  ALM_REQUIRE(kind != ALM_MODEL_OMNI_SPOT || m->vie == 0, ALM_ERR_INVALID, "text-spotting checkpoint must have V = 1104");
  m->word_emb = upload_f32(c, we.f32.data(), we.numel());
  const char* kinds[3] = {"pt", "poly", "rec"};
  for (int d = 0; d < 3; ++d) {
    const HostTensor& pe = need(t, tr + "embedding." + kinds[d] + "_position_embeddings.weight");
    ALM_REQUIRE(pe.numel() == size_t(1024) * 512, ALM_ERR_INVALID, "position embedding shape");
    m->pos_emb[d] = upload_f32(c, pe.f32.data(), pe.numel());
  }
  m->emb_norm = load_ln(c, t, tr + "embedding.LayerNorm", 512);
  std::vector<float> kw(size_t(12) * 512 * 512), kb(12 * 512), vw(size_t(12) * 512 * 512), vb(12 * 512);
  for (int d = 0; d < 3; ++d) {
    for (int l = 0; l < 4; ++l) {
      const std::string p = tr + kinds[d] + "_decoder.layers." + std::to_string(l) + ".";
      DecLayerW& w = m->dec[d][l];
      w.n1 = load_ln(c, t, p + "norm1", 512);
      w.n2 = load_ln(c, t, p + "norm2", 512);
      w.n3 = load_ln(c, t, p + "norm3", 512);
      {
        const HostTensor& ipw0 = need(t, p + "self_attn.in_proj_weight");
        const HostTensor& ipb0 = need(t, p + "self_attn.in_proj_bias");
        w.sa_qkv_f = upload_f32(c, ipw0.f32.data(), ipw0.numel());
        w.sa_qkv_b = upload_f32(c, ipb0.f32.data(), ipb0.numel());
      }
      if (d == 0) {  // the polygon / recognition decoders' linears are loaded in pairs below
        w.sa_qk = load_inproj_rows(c, t, p + "self_attn", 0, 1024);
        w.sa_v = load_inproj_rows(c, t, p + "self_attn", 1024, 512);
        w.sa_out = load_lin(c, t, p + "self_attn.out_proj", 512, 512, true, 0, true);
        w.ca_q = load_inproj_rows(c, t, p + "multihead_attn", 0, 512);
        w.ca_out = load_lin(c, t, p + "multihead_attn.out_proj", 512, 512, true, 0, true);
        w.l1 = load_lin(c, t, p + "linear1", 2048, 512, true, 0, true);
        w.l2 = load_lin(c, t, p + "linear2", 512, 2048, true, 0, true);
      }
      const HostTensor& ipw = need(t, p + "multihead_attn.in_proj_weight");
      const HostTensor& ipb = need(t, p + "multihead_attn.in_proj_bias");
      const size_t dl = static_cast<size_t>(d) * 4 + l;
      std::copy(ipw.f32.begin() + size_t(512) * 512, ipw.f32.begin() + size_t(1024) * 512, kw.begin() + dl * 512 * 512);
      std::copy(ipw.f32.begin() + size_t(1024) * 512, ipw.f32.begin() + size_t(1536) * 512, vw.begin() + dl * 512 * 512);
      std::copy(ipb.f32.begin() + 512, ipb.f32.begin() + 1024, kb.begin() + dl * 512);
      std::copy(ipb.f32.begin() + 1024, ipb.f32.begin() + 1536, vb.begin() + dl * 512);
    }
    m->dec_norm[d] = load_ln(c, t, tr + kinds[d] + "_decoder.norm", 512);
    if (d == 0) {
      const std::string hp = tr + kinds[d] + "_pred_layer.layers.";
      m->head[d][0] = load_lin(c, t, hp + "0", 512, 512, true, 0, true);
      m->head[d][1] = load_lin(c, t, hp + "1", 512, 512, true, 0, true);
      m->head[d][2] = load_lin(c, t, hp + "2", m->V, 512, true, 0, true);
    }
  }
  // polygon + recognition decoders: every linear of decoder 2 sits one weight further along decoder 1's slab, so the
  // joint decoder pass runs each of them as one GEMM over both decoders' rows
  for (int l = 0; l < 4; ++l) {
    const std::string lp[2] = {tr + "poly_decoder.layers." + std::to_string(l) + ".",
                               tr + "rec_decoder.layers." + std::to_string(l) + "."};
    auto pair = [&](const std::string& suffix, int N, int K, bool inproj, int r0, Lin DecLayerW::*f) {
      const std::string p[2] = {lp[0] + suffix, lp[1] + suffix};
      Lin out[2];
      load_lin_pair(c, t, p, N, K, inproj, r0, out);
      m->dec[1][l].*f = out[0];
      m->dec[2][l].*f = out[1];
    };
    pair("self_attn", 1024, 512, true, 0, &DecLayerW::sa_qk);
    pair("self_attn", 512, 512, true, 1024, &DecLayerW::sa_v);
    pair("self_attn.out_proj", 512, 512, false, 0, &DecLayerW::sa_out);
    pair("multihead_attn", 512, 512, true, 0, &DecLayerW::ca_q);
    pair("multihead_attn.out_proj", 512, 512, false, 0, &DecLayerW::ca_out);
    pair("linear1", 2048, 512, false, 0, &DecLayerW::l1);
    pair("linear2", 512, 2048, false, 0, &DecLayerW::l2);
  }
  for (int k = 0; k < 3; ++k) {
    const std::string p[2] = {tr + "poly_pred_layer.layers." + std::to_string(k),
                              tr + "rec_pred_layer.layers." + std::to_string(k)};
    Lin out[2];
    load_lin_pair(c, t, p, k == 2 ? m->V : 512, 512, false, 0, out);
    m->head[1][k] = out[0];
    m->head[2][k] = out[1];
  }
  m->ca_k_all.w = upload_split(c, kw.data(), 12 * 512, 512, 0);
  m->ca_k_all.b = upload_f32(c, kb.data(), kb.size());
  m->ca_v_all.w = upload_split(c, vw.data(), 12 * 512, 512, 0);
  m->ca_v_all.b = upload_f32(c, vb.data(), vb.size());
  delete c->omni;
  c->omni = m;
}

OmniModel* omni_share(const OmniModel* owner) {
  OmniModel* m = new OmniModel(*owner);  // weight pointers (the slabs are ref-counted by Ctx::wstore)
  m->step_graphs.clear();                // graphs, encode state and cache pointers belong to the owner's arena
  m->encoded = false;
  m->B = m->H = m->W = m->M = m->Mpad = m->mh = m->mw = 0;
  for (auto& f : m->feat) f = nullptr;
  m->memory = m->pos = nullptr;
  m->kpm = nullptr;
  m->kc_hi = m->kc_lo = m->vc_hi = m->vc_lo = m->vt_hi = m->vt_lo = nullptr;
  m->page_mh.clear(); m->page_mw.clear(); m->page_keys.clear();
  m->rec_lists = {};
  m->dense_loops.clear();
  m->mixed = false;
  m->key_len = m->kb_off = nullptr;
  m->d_page_mw = nullptr;
  m->ws_mark = 0;
  return m;
}

std::vector<float> sine_dim_t() {
  std::vector<float> dt(256);
  for (int i = 0; i < 256; ++i) dt[i] = powf(10000.0f, (2.0f * static_cast<float>(i / 2)) / 256.0f);
  return dt;
}

// ================================================================================================ encode
void stage_grid(int H, int W, int* Hs, int* Ws) {
  int hs = (H + 3) / 4, wsz = (W + 3) / 4;
  for (int s = 0; s < 4; ++s) {
    Hs[s] = hs; Ws[s] = wsz;
    hs = (hs + 1) / 2; wsz = (wsz + 1) / 2;
  }
}

namespace {

// Swin-B -> FPN -> input_proj of B images of one size H x W, read from the canvas slots `slots` (NULL: slot b) of
// img [*, 3, Hc, Wc].  feat: the persistent stage outputs, or NULL (not kept).  mem_map: memory row of each of the
// B * mh * mw output rows (NULL: in order).  Every activation is allocated after `mark` and released on return.
void encode_group(Ctx* c, OmniModel* m, const float* img, int Hc, int Wc, const int* slots, int B, int H, int W,
                  float* const* feat, const int* mem_map) {
  Arena& ws = c->ws;
  const size_t group_mark = ws.mark();
  int Hs[4], Ws[4];
  stage_grid(H, W, Hs, Ws);
  const int mh = Hs[2], mw = Ws[2];
  const long BM = static_cast<long>(B) * mh * mw;

  // ---- patch embed: im2col -> GEMM(+bias) -> LN   (swin_transformer.py:427-443)
  long rows = static_cast<long>(B) * Hs[0] * Ws[0];
  float* x = ws.get<float>(rows * 128);
  {
    const size_t mk = ws.mark();
    SplitBuf a = alloc_split(c, rows * 64);
    float* tmp = ws.get<float>(rows * 128);
    im2col_patch4(c, img, B, H, W, Hs[0], Ws[0], a.hi, a.lo, Hc, Wc, slots);
    linear(c, a, rows, m->patch, ACT_NONE, tmp, nullptr);
    gather_ln(c, tmp, 128, nullptr, 1, 128, rows, m->patch_norm.g, m->patch_norm.b, 1e-5f, false, nullptr, 0, x, 128,
              nullptr, nullptr, 0, nullptr, nullptr);
    ws.release(mk);
    // x was allocated before mk, tmp/a are dead after the LN (stream-ordered)
  }

  SplitBuf feat_split[4];
  for (int s = 0; s < 4; ++s) {
    const int C = 128 << s, heads = kHeads[s];
    const int Hc_ = Hs[s], Wc_ = Ws[s];
    const int nWh = (Hc_ + 6) / 7, nWw = (Wc_ + 6) / 7;
    const long rowsP = static_cast<long>(B) * nWh * nWw * 49;
    rows = static_cast<long>(B) * Hc_ * Wc_;
    const size_t stage_mark = ws.mark();
    int* map0 = ws.get<int>(rowsP);
    int* map1 = ws.get<int>(rowsP);
    window_map(c, map0, B, Hc_, Wc_, nWh, nWw, 0);
    window_map(c, map1, B, Hc_, Wc_, nWh, nWw, 3);
    SplitBuf lnw = alloc_split(c, std::max(rowsP, rows) * C);
    SplitBuf qkv = alloc_split(c, rowsP * 3 * C);
    SplitBuf att = alloc_split(c, rowsP * C);
    SplitBuf hid = alloc_split(c, rows * 4 * C);
    for (int b = 0; b < kDepths[s]; ++b) {
      const SwinBlockW& w = m->stage[s].blocks[b];
      const int shift = (b & 1) ? 3 : 0;
      const int* map = shift ? map1 : map0;
      // LN1 -> zero-pad -> roll -> window partition, as one gather (pad tokens stay live keys, F10)
      gather_ln(c, x, C, map, 1, C, rowsP, w.n1.g, w.n1.b, 1e-5f, true, nullptr, 0, nullptr, 0, lnw.hi, lnw.lo, C,
                nullptr, nullptr);
      linear(c, lnw, rowsP, w.qkv, ACT_NONE, nullptr, &qkv);
      window_attention_split(c, qkv.hi, qkv.lo, C, heads, nWh, nWw, B, shift, nWh * 7, nWw * 7, w.bias_dense, att.hi,
                             att.lo, nullptr);
      // proj + window reverse + un-roll + crop + residual, fused in the GEMM epilogue (scatter map)
      linear(c, att, rowsP, w.proj, ACT_NONE, x, nullptr, x, map, nullptr, C);
      gather_ln(c, x, C, nullptr, 1, C, rows, w.n2.g, w.n2.b, 1e-5f, false, nullptr, 0, nullptr, 0, lnw.hi, lnw.lo, C,
                nullptr, nullptr);
      linear(c, lnw, rows, w.fc1, ACT_GELU, nullptr, &hid);
      linear(c, hid, rows, w.fc2, ACT_NONE, x, nullptr, x, nullptr, nullptr, C);
    }
    ws.release(stage_mark);
    // per-stage output norm (swin_transformer.py:616-618): fp32 feature (API) + split operand (FPN)
    feat_split[s] = alloc_split(c, rows * C);
    gather_ln(c, x, C, nullptr, 1, C, rows, m->stage[s].out_norm.g, m->stage[s].out_norm.b, 1e-5f, false, nullptr, 0,
              feat ? feat[s] : nullptr, C, feat_split[s].hi, feat_split[s].lo, C, nullptr, nullptr);
    if (s < 3) {
      // PatchMerging: 2x2 gather-concat -> LN(4C) -> Linear 4C->2C (swin_transformer.py:269-296)
      const int H2 = Hs[s + 1], W2 = Ws[s + 1];
      const long rows2 = static_cast<long>(B) * H2 * W2;
      float* xn = ws.get<float>(rows2 * 2 * C);
      const size_t mk = ws.mark();
      int* mm = ws.get<int>(rows2 * 4);
      SplitBuf ma = alloc_split(c, rows2 * 4 * C);
      merge_map(c, mm, B, Hc_, Wc_, H2, W2);
      gather_ln(c, x, C, mm, 4, C, rows2, m->stage[s].merge_norm.g, m->stage[s].merge_norm.b, 1e-5f, false, nullptr, 0,
                nullptr, 0, ma.hi, ma.lo, 4 * C, nullptr, nullptr);
      Lin red;
      red.w = m->stage[s].merge_red;
      linear(c, ma, rows2, red, ACT_NONE, xn, nullptr);
      ws.release(mk);
      x = xn;
    }
  }

  // ---- FPN (fpn.py:21-45): p5, p4 = c4' + up(p5), p3, p2 at full resolution, fp32
  float* p[4];  // p[0]=p2 (stage 0 res) ... p[3]=p5
  for (int s = 0; s < 4; ++s) p[s] = ws.get<float>(static_cast<size_t>(B) * Hs[s] * Ws[s] * 256);
  for (int s = 3; s >= 0; --s) {
    rows = static_cast<long>(B) * Hs[s] * Ws[s];
    Lin l;
    l.w = m->fpn[3 - s];
    if (s == 3) {
      linear(c, feat_split[s], rows, l, ACT_NONE, p[s], nullptr);
    } else {
      const size_t mk = ws.mark();
      int* up = ws.get<int>(rows);
      nearest_map(c, up, B, Hs[s], Ws[s], Hs[s + 1], Ws[s + 1]);
      linear(c, feat_split[s], rows, l, ACT_NONE, p[s], nullptr, p[s + 1], nullptr, up, 256);
      ws.release(mk);  // map is consumed by the GEMM already enqueued; later allocations are stream-ordered after it
    }
  }
  // consumer-side assembly of the stride-2-sampled concat + input_proj (omniparser.py:15,31); the GEMM epilogue
  // scatters each page's rows to its memory slot
  SplitBuf cat = alloc_split(c, BM * 1024);
  fpn_assemble(c, p[0], p[1], p[2], p[3], B, Hs, Ws, mh, mw, cat.hi, cat.lo);
  linear(c, cat, BM, m->inproj, ACT_NONE, m->memory, nullptr, nullptr, mem_map);
  ws.release(group_mark);
}

struct PageGroup {
  int h, w;
  std::vector<int> slots;
};

// heights / widths NULL: B images of H x W with an optional padding mask (alm_omni_encode).  Otherwise the pages are
// encoded per size group, each page on its own grid without a mask; one group leaves the state of alm_omni_encode.
void encode_impl(Ctx* c, const float* img, const uint8_t* mask, int B, int H, int W, const int* heights,
                 const int* widths) {
  OmniModel* m = c->omni;
  Arena& ws = c->ws;
  ws.off = 0;
  m->encoded = false;
  struct CapGuard {
    Ctx* c;
    ~CapGuard() { c->gemm_grid_cap = 0; }
  } cap_guard{c};
  c->gemm_grid_cap = c->enc_grid_cap;
  if (!c->ev_t[0]) for (auto& e : c->ev_t) ALM_CHECK_CUDA(cudaEventCreate(&e));
  ALM_CHECK_CUDA(cudaEventRecord(c->ev_t[0], c->stream));
  m->B = B; m->H = H; m->W = W;

  std::vector<PageGroup> groups;  // size groups in order of first appearance
  m->page_mh.assign(B, 0);
  m->page_mw.assign(B, 0);
  for (int b = 0; b < B; ++b) {
    const int h = heights ? heights[b] : H, w = widths ? widths[b] : W;
    auto g = std::find_if(groups.begin(), groups.end(), [&](const PageGroup& x) { return x.h == h && x.w == w; });
    if (g == groups.end()) g = groups.insert(groups.end(), PageGroup{h, w, {}});
    g->slots.push_back(b);
    int Hs[4], Ws[4];
    stage_grid(h, w, Hs, Ws);
    m->page_mh[b] = Hs[2];
    m->page_mw[b] = Ws[2];
  }
  m->mixed = groups.size() > 1;
  m->page_keys.clear();
  if (!m->mixed) {
    stage_grid(groups[0].h, groups[0].w, m->Hs, m->Ws);
    m->mh = m->Hs[2]; m->mw = m->Ws[2];
    m->M = m->mh * m->mw;
  } else {
    for (int s = 0; s < 4; ++s) m->Hs[s] = m->Ws[s] = 0;
    m->mh = m->mw = 0;
    for (int b = 0; b < B; ++b) m->page_keys.push_back(m->page_mh[b] * m->page_mw[b]);
    m->M = *std::max_element(m->page_keys.begin(), m->page_keys.end());
  }
  m->Mpad = (m->M + 7) & ~7;
  const long BM = static_cast<long>(B) * m->M;

  // ---- encode-persistent buffers (memory rows of page b at b * M)
  for (int s = 0; s < 4; ++s)
    m->feat[s] = m->mixed ? nullptr : ws.get<float>(static_cast<size_t>(B) * m->Hs[s] * m->Ws[s] * (128 << s));
  m->memory = ws.get<float>(BM * 512);
  m->pos = ws.get<float>(BM * 512);
  m->kpm = ws.get<uint8_t>(BM);
  m->kc_hi = ws.get<bf16>(BM * 6144);
  m->kc_lo = ws.get<bf16>(BM * 6144);
  m->vc_hi = ws.get<bf16>(BM * 6144);
  m->vc_lo = ws.get<bf16>(BM * 6144);
  m->vt_hi = m->vt_lo = nullptr;
  if (c->xattn_impl == 1) {  // the unfused debug path multiplies P by a feature-major V_c^T
    m->vt_hi = ws.get<bf16>(static_cast<size_t>(B) * 6144 * m->Mpad);
    m->vt_lo = ws.get<bf16>(static_cast<size_t>(B) * 6144 * m->Mpad);
  }
  m->key_len = m->kb_off = nullptr;
  std::vector<int> h_idx;  // mixed: key_len [B], kb_off [B + 1], then per group its slots and memory row map
  if (m->mixed) {
    m->key_len = ws.get<int>(2 * B + 1);
    m->kb_off = m->key_len + B;
    h_idx = m->page_keys;
    h_idx.push_back(0);
    for (int b = 0; b < B; ++b) h_idx.push_back(h_idx.back() + (m->page_keys[b] + 63) / 64);
  }
  // grid width of every page: the key -> position map of the character locations
  m->d_page_mw = ws.get<int>(B);
  ALM_CHECK_CUDA(cudaMemcpyAsync(m->d_page_mw, m->page_mw.data(), B * sizeof(int), cudaMemcpyHostToDevice, c->stream));
  m->ws_mark = ws.mark();

  if (!m->mixed) {
    encode_group(c, m, img, H, W, nullptr, B, groups[0].h, groups[0].w, m->feat, nullptr);
    float* scratch = ws.get<float>(static_cast<size_t>(2) * BM);
    sine_pos(c, mask, B, groups[0].h, groups[0].w, m->mh, m->mw, m->dim_t, m->pos, m->kpm, scratch);
  } else {
    std::vector<size_t> gofs;
    for (const PageGroup& g : groups) {
      gofs.push_back(h_idx.size());
      h_idx.insert(h_idx.end(), g.slots.begin(), g.slots.end());
      const int Mg = m->page_keys[g.slots[0]];
      for (int slot : g.slots)
        for (int r = 0; r < Mg; ++r) h_idx.push_back(slot * m->M + r);
    }
    int* d_idx = ws.get<int>(h_idx.size());
    ALM_CHECK_CUDA(cudaMemcpyAsync(d_idx, h_idx.data(), h_idx.size() * sizeof(int), cudaMemcpyHostToDevice, c->stream));
    ALM_CHECK_CUDA(cudaMemcpyAsync(m->key_len, d_idx, (2 * B + 1) * sizeof(int), cudaMemcpyDeviceToDevice, c->stream));
    // rows beyond a page's keys: zero memory / pos, masked keys
    ALM_CHECK_CUDA(cudaMemsetAsync(m->memory, 0, BM * 512 * sizeof(float), c->stream));
    ALM_CHECK_CUDA(cudaMemsetAsync(m->pos, 0, BM * 512 * sizeof(float), c->stream));
    ALM_CHECK_CUDA(cudaMemsetAsync(m->kpm, 1, BM, c->stream));
    const size_t groups_mark = ws.mark();
    for (size_t gi = 0; gi < groups.size(); ++gi) {
      const PageGroup& g = groups[gi];
      const int Bg = static_cast<int>(g.slots.size());
      const int* slots = d_idx + gofs[gi];
      encode_group(c, m, img, H, W, slots, Bg, g.h, g.w, nullptr, slots + Bg);
      // every page of the group has the same unmasked position embedding: computed once, copied to each slot
      const int mh = m->page_mh[g.slots[0]], mw = m->page_mw[g.slots[0]], Mg = mh * mw;
      float* pos1 = ws.get<float>(static_cast<size_t>(Mg) * 512);
      uint8_t* kpm1 = ws.get<uint8_t>(Mg);
      float* scratch = ws.get<float>(static_cast<size_t>(2) * Mg);
      sine_pos(c, nullptr, 1, g.h, g.w, mh, mw, m->dim_t, pos1, kpm1, scratch);
      for (int slot : g.slots) {
        const long r0 = static_cast<long>(slot) * m->M;
        ALM_CHECK_CUDA(cudaMemcpyAsync(m->pos + r0 * 512, pos1, static_cast<size_t>(Mg) * 512 * sizeof(float),
                                       cudaMemcpyDeviceToDevice, c->stream));
        ALM_CHECK_CUDA(cudaMemsetAsync(m->kpm + r0, 0, Mg, c->stream));
      }
      ws.release(groups_mark);
    }
  }
  // operands for the cross-attention K/V projections: memory and memory + pos
  SplitBuf mem = alloc_split(c, BM * 512), memp = alloc_split(c, BM * 512);
  gather_ln(c, m->memory, 512, nullptr, 1, 512, BM, nullptr, nullptr, 0.f, false, m->pos, 512, nullptr, 0, mem.hi,
            mem.lo, 512, memp.hi, memp.lo);
  {  // K_c[b][dl][h][m][64] = (memory + pos) Wk^T + bk for all 12 (decoder, layer) pairs: head-major so that the keys
     // of one (image, layer, head) are one contiguous 128-byte-row block (the per-token decode streams exactly that)
    Operand a = act_op(memp.hi, memp.lo, m->M, 512, 512);
    a.nb1 = B; a.bs1 = static_cast<long>(m->M) * 512;
    Operand w = m->ca_k_all.w.op();
    w.rows = 512; w.nb0 = 4 * c->kv_decoders; w.bs0 = static_cast<long>(512) * 512;  // (decoder, layer) slices, 8 heads wide
    Epilogue e;
    e.out_hi = m->kc_hi; e.out_lo = m->kc_lo; e.ldo = 64;
    e.obs0 = static_cast<long>(8) * m->M * 64; e.obs1 = static_cast<long>(96) * m->M * 64;
    e.col_group = 64; e.col_group_stride = static_cast<long>(m->M) * 64;  // head h = column / 64 -> its own [M, 64] block
    e.bias = m->ca_k_all.b; e.bias_mode = BIAS_COL; e.bias_bs0 = 512;
    gemm(c, a, w, e);
  }
  {  // V_c[b][dl][h][m][64] = memory Wv^T + bv, same head-major layout: a 64-key block of one (image, layer, head) is
     // one contiguous 8 KB run per plane, which is what the fused attention streams
    Operand a = act_op(mem.hi, mem.lo, m->M, 512, 512);
    a.nb1 = B; a.bs1 = static_cast<long>(m->M) * 512;
    Operand w = m->ca_v_all.w.op();
    w.rows = 512; w.nb0 = 4 * c->kv_decoders; w.bs0 = static_cast<long>(512) * 512;
    Epilogue e;
    e.out_hi = m->vc_hi; e.out_lo = m->vc_lo; e.ldo = 64;
    e.obs0 = static_cast<long>(8) * m->M * 64; e.obs1 = static_cast<long>(96) * m->M * 64;
    e.col_group = 64; e.col_group_stride = static_cast<long>(m->M) * 64;
    e.bias = m->ca_v_all.b; e.bias_mode = BIAS_COL; e.bias_bs0 = 512;
    gemm(c, a, w, e);
  }
  if (m->vt_hi) {  // V_c^T[b, dl*512 + f, m] = Wv memory^T + bv  (feature-major so that P.V is a K-major GEMM)
    Operand bop = act_op(mem.hi, mem.lo, m->M, 512, 512);
    bop.nb1 = B; bop.bs1 = static_cast<long>(m->M) * 512;
    Epilogue e;
    e.out_hi = m->vt_hi; e.out_lo = m->vt_lo; e.ldo = m->Mpad; e.obs1 = static_cast<long>(6144) * m->Mpad;
    e.bias = m->ca_v_all.b; e.bias_mode = BIAS_ROW;
    gemm(c, m->ca_v_all.w.op(), bop, e);
  }
  ws.release(m->ws_mark);
  m->encoded = true;
  m->kv_decoders = c->kv_decoders;
  ALM_CHECK_CUDA(cudaEventRecord(c->ev_t[1], c->stream));
  c->timing_valid[0] = true;
}

}  // namespace

void omni_encode(Ctx* c, const float* img, const uint8_t* mask, int B, int H, int W) {
  ALM_REQUIRE(c->omni != nullptr, ALM_ERR_STATE, "alm_omni_encode before alm_load_weights");
  ALM_REQUIRE(B > 0 && H >= 32 && W >= 32, ALM_ERR_INVALID, "image batch must be non-empty and at least 32x32");
  c->ensure_ws();
  encode_impl(c, img, mask, B, H, W, nullptr, nullptr);
}

void omni_encode_pages(Ctx* c, const float* img, int B, int Hc, int Wc, const int* heights, const int* widths) {
  ALM_REQUIRE(c->omni != nullptr, ALM_ERR_STATE, "alm_omni_encode_pages before alm_load_weights");
  ALM_REQUIRE(B > 0, ALM_ERR_INVALID, "page batch must be non-empty");
  for (int b = 0; b < B; ++b)
    ALM_REQUIRE(heights[b] >= 32 && widths[b] >= 32 && heights[b] <= Hc && widths[b] <= Wc, ALM_ERR_INVALID,
                "page " + std::to_string(b) + " must be at least 32x32 and fit the canvas");
  c->ensure_ws();
  encode_impl(c, img, nullptr, B, Hc, Wc, heights, widths);
}

// ================================================================================================ decode
namespace {

using Points = std::vector<std::pair<int, int>>;

struct DecodeBufs {
  int S = 0, Tmax = 0, Ncap = 0;
  float* x = nullptr;
  float* qpos = nullptr;  // [512] query_pos of the current step
  int* tpos = nullptr;    // device-side position counter (so one captured graph serves every token)
  SplitBuf ln, lnp, att, q, o, hid, h0, h1;
  float *qk = nullptr, *v = nullptr, *scores = nullptr, *logits = nullptr, *qf = nullptr;
  float* qkv = nullptr;  // skinny path: fused [S,1536] q|k|v
  float *lnf = nullptr, *lnpf = nullptr, *attf = nullptr, *of = nullptr, *hidf = nullptr, *h0f = nullptr, *h1f = nullptr;
  bool skinny = false;          // S <= 32 live sequences: all-fp32 SIMT GEMV path instead of tensor-core tiles
  float* xq_partial = nullptr;  // fused single-query cross-attention: split partials + counters
  int* xq_counters = nullptr;
  int xq_splits = 1;
  int mq_grid = 1, mq_parts = 1;  // fused cross-attention: persistent grid size, partial slots per (image, head, query block)
  bool fused_xattn = false;
  bool tma_xattn = false;  // fused, TMA + mbarrier variant of the mma.sync kernel (xattn_impl 2)
  SplitBuf prob;
  float* kc[4] = {nullptr, nullptr, nullptr, nullptr};
  float* vc[4] = {nullptr, nullptr, nullptr, nullptr};
  const int* anc = nullptr;  // beam search: [S][Tmax] row holding each cached position of each sequence (NULL: its own)
  // rec loop with character locations: [S][loc_L][5] (NULL: off), the locate kernel's key splits, partials, counters
  float* loc = nullptr;
  int loc_L = 0, loc_ks = 1;
  float* loc_partial = nullptr;
  int* loc_counters = nullptr;
};

// The rows of nd decoders d0 .. d0 + nd - 1 stepped together, and each decoder's rows as single-decoder buffers (its
// head selection, its cross-attention, the steps its loop runs alone).  nd 2 is the joint polygon + recognition pass:
// rows [0, S) are the polygon sequences, rows [S, 2S) the recognition sequences.  With nd 1 the view is the rows.
struct StepBufs {
  int nd = 1;
  DecodeBufs all, half[2];
  DecodeBufs& v(int i) { return nd == 1 ? all : half[i]; }
};

// nd decoders x B images x Ncap sequences each, caches of Tmax positions (nd 2: the longer loop's, for both halves).
// pt_loop: the point loop may take the skinny path with up to 16 prompts per image (the fused cross-attention serves
// them as the rows of its 16-query variant); the poly / rec loops and teacher forcing take it with one sequence per image.
// img0: first image of the B the buffers serve (its live-key counts size the cross-attention schedule)
StepBufs alloc_decode(Ctx* c, OmniModel* m, int nd, int B, int Ncap, int Tmax, bool pt_loop, int img0) {
  StepBufs sb;
  sb.nd = nd;
  DecodeBufs& d = sb.all;
  const size_t S = static_cast<size_t>(B) * Ncap, R = nd * S;  // rows per decoder, rows in all
  d.S = static_cast<int>(R); d.Tmax = Tmax; d.Ncap = Ncap;
  d.x = c->ws.get<float>(R * 512);
  d.qpos = c->ws.get<float>(nd * 512);
  d.tpos = c->ws.get<int>(1);
  d.ln = alloc_split(c, R * 512);
  d.lnp = alloc_split(c, R * 512);
  d.att = alloc_split(c, R * 512);
  d.q = alloc_split(c, R * 512);
  d.o = alloc_split(c, R * 512);
  d.hid = alloc_split(c, R * 2048);
  d.h0 = alloc_split(c, R * 512);
  d.h1 = alloc_split(c, R * 512);
  d.qk = c->ws.get<float>(R * 1024);
  d.v = c->ws.get<float>(R * 512);
  d.qf = c->ws.get<float>(R * 512);
  d.logits = c->ws.get<float>(R * m->V);
  for (int l = 0; l < 4; ++l) {
    d.kc[l] = c->ws.get<float>(R * Tmax * 512);
    d.vc[l] = c->ws.get<float>(R * Tmax * 512);
  }
  // xattn_impl 1 has a one-query skinny kernel only (cross_attn_q1); the joint pass has no skinny step
  d.skinny = nd == 1 && S <= 32 && (Ncap == 1 || (pt_loop && Ncap <= 16 && c->xattn_impl != 1));
  if (d.skinny) {
    d.lnf = c->ws.get<float>(S * 512); d.lnpf = c->ws.get<float>(S * 512); d.attf = c->ws.get<float>(S * 512);
    d.of = c->ws.get<float>(S * 512); d.hidf = c->ws.get<float>(S * 2048); d.h0f = c->ws.get<float>(S * 512);
    d.h1f = c->ws.get<float>(S * 512);
    d.qkv = c->ws.get<float>(S * 1536);
  }
  for (int i = 0; i < nd; ++i) {
    DecodeBufs& u = sb.v(i);
    if (nd > 1) {  // decoder i's rows [i S, (i + 1) S) of every buffer
      const size_t r = i * S;
      auto rows = [&](const SplitBuf& b, size_t w) { return SplitBuf{b.hi + r * w, b.lo + r * w}; };
      u = d;
      u.S = static_cast<int>(S);
      u.x = d.x + r * 512;
      u.qpos = d.qpos + i * 512;
      u.ln = rows(d.ln, 512); u.lnp = rows(d.lnp, 512); u.att = rows(d.att, 512); u.q = rows(d.q, 512);
      u.o = rows(d.o, 512); u.hid = rows(d.hid, 2048); u.h0 = rows(d.h0, 512); u.h1 = rows(d.h1, 512);
      u.qk = d.qk + r * 1024;
      u.v = d.v + r * 512;
      u.qf = d.qf + r * 512;
      u.logits = d.logits + r * m->V;
      for (int l = 0; l < 4; ++l) {
        u.kc[l] = d.kc[l] + r * Tmax * 512;
        u.vc[l] = d.vc[l] + r * Tmax * 512;
      }
    }
    // the decoder's own cross-attention schedule: the fused kernels' plan, partials and counters, the one-query
    // kernel's key splits, or the unfused path's score and probability planes
    if (c->xattn_impl == 0 || c->xattn_impl == 2) {
      int pairs = 0;
      u.fused_xattn = true;
      u.tma_xattn = c->xattn_impl == 2;
      const int* key_len = m->mixed ? m->page_keys.data() + img0 : nullptr;
      if (u.tma_xattn) cross_attn_tma_plan(c, B, Ncap, m->M, &u.mq_grid, &u.mq_parts, &pairs, key_len);
      else cross_attn_mq_plan(c, B, Ncap, m->M, &u.mq_grid, &u.mq_parts, &pairs, key_len);
      u.xq_partial = c->ws.get<float>(cross_attn_mq_partial_floats(pairs, u.mq_parts));
      u.xq_counters = c->ws.get<int>(pairs);
      fill_i32(c, u.xq_counters, pairs, 0);
    } else if (Ncap == 1) {
      u.xq_splits = cross_attn_q1_splits(c, B, m->M);
      u.xq_partial = c->ws.get<float>(static_cast<size_t>(B) * 8 * u.xq_splits * 66);
      u.xq_counters = c->ws.get<int>(static_cast<size_t>(B) * 8);
      fill_i32(c, u.xq_counters, static_cast<long>(B) * 8, 0);
    } else {
      u.scores = c->ws.get<float>(S * 8 * m->Mpad);
      u.prob = alloc_split(c, S * 8 * m->Mpad);
    }
  }
  return sb;
}

// Fused cross-attention of `nimg` images x Ncap queries against decoder-layer dl of the cached K_c / V_c
void fused_xattn(Ctx* c, OmniModel* m, DecodeBufs& u, const bf16* q_hi, const bf16* q_lo, const float* q_f32, int img0, int nimg,
                 int Ncap, long dl, bf16* out_hi, bf16* out_lo, float* out_f32) {
  const int M = m->M;
  const uint8_t* kpm = m->kpm + static_cast<long>(img0) * M;
  // pages of different sizes: only each page's own key blocks are streamed
  const int* key_len = m->key_len ? m->key_len + img0 : nullptr;
  const int* kb_off = m->kb_off ? m->kb_off + img0 : nullptr;
  if (u.tma_xattn) {
    cross_attn_tma(c, q_hi, q_lo, q_f32, nimg, Ncap, m->kc_hi, m->kc_lo, m->vc_hi, m->vc_lo, static_cast<long>(m->B) * 96,
                   static_cast<int>(img0 * 96 + dl * 8), kpm, M, key_len, kb_off, u.mq_grid, u.mq_parts, u.xq_partial,
                   u.xq_counters, out_hi, out_lo, out_f32);
    return;
  }
  const long koff = (static_cast<long>(img0) * 96 + dl * 8) * M * 64;
  cross_attn_mq(c, q_hi, q_lo, q_f32, nimg, Ncap, m->kc_hi + koff, m->kc_lo + koff, m->vc_hi + koff, m->vc_lo + koff, kpm, M,
                key_len, kb_off, u.mq_grid, u.mq_parts, u.xq_partial, u.xq_counters, out_hi, out_lo, out_f32);
}

// Character locations of a generated rec step: the last layer's cross-attention queries (split or fp32) against its
// K cache, reduced to moments at step *u.tpos - 2 (the rec prompt is [x, y, sos]).
void rec_locate_step(Ctx* c, OmniModel* m, DecodeBufs& u, const bf16* q_hi, const bf16* q_lo, const float* q_f32,
                     int img0, int nimg) {
  const long koff = (static_cast<long>(img0) * 96 + 11 * 8) * m->M * 64;
  rec_locate(c, q_hi, q_lo, q_f32, nimg, u.Ncap, m->kc_hi + koff, m->kc_lo + koff, m->kpm + static_cast<long>(img0) * m->M,
             m->M, m->key_len ? m->key_len + img0 : nullptr, m->d_page_mw + img0, u.loc_ks, u.loc_partial, u.loc_counters,
             u.tpos, 2, u.loc_L, u.loc);
}

// The cross-attention of one decoder's rows `u` against decoder layer dl (d * 4 + l) of the cached K_c / V_c^T of
// images img0 .. img0 + nimg - 1.  Queries in qf (fp32) on the skinny step or with one query per image, else in the
// split planes q; the output to of (fp32) on the skinny step, else to the split planes o.  A generated rec step with
// locations on also hands the last layer's queries to the locate kernel.
void cross_attn(Ctx* c, OmniModel* m, DecodeBufs& u, long dl, int img0, int nimg, bool want_logits) {
  const int M = m->M, Mpad = m->Mpad, Ncap = u.Ncap;
  const bool q32 = u.skinny || Ncap == 1;
  const bf16 *q_hi = q32 ? nullptr : u.q.hi, *q_lo = q32 ? nullptr : u.q.lo;
  const float* q_f32 = q32 ? u.qf : nullptr;
  bf16 *o_hi = u.skinny ? nullptr : u.o.hi, *o_lo = u.skinny ? nullptr : u.o.lo;
  float* o_f32 = u.skinny ? u.of : nullptr;
  if (u.loc && want_logits && dl == 11) rec_locate_step(c, m, u, q_hi, q_lo, q_f32, img0, nimg);
  if (u.fused_xattn) {
    // scores, mask, online softmax and P.V fused; K_c / V_c streamed once per layer-step (HBM-bound)
    fused_xattn(c, m, u, q_hi, q_lo, q_f32, img0, nimg, Ncap, dl, o_hi, o_lo, o_f32);
    return;
  }
  const long koff = (static_cast<long>(img0) * 96 + dl * 8) * M * 64;
  const long voff = (static_cast<long>(img0) * 6144 + dl * 512) * Mpad;
  if (Ncap == 1) {
    cross_attn_q1(c, u.qf, m->kc_hi + koff, m->kc_lo + koff, m->vt_hi + voff, m->vt_lo + voff,
                  m->kpm + static_cast<long>(img0) * M, nimg, M, Mpad, u.xq_partial, u.xq_counters, u.xq_splits, o_hi,
                  o_lo, o_f32);
    return;
  }
  {
    Operand a = act_op(u.q.hi, u.q.lo, Ncap, 64, 512);
    a.nb0 = 8; a.bs0 = 64; a.nb1 = nimg; a.bs1 = static_cast<long>(Ncap) * 512;
    Operand k = act_op(m->kc_hi + koff, m->kc_lo + koff, M, 64, 64);
    k.nb0 = 8; k.bs0 = static_cast<long>(M) * 64; k.nb1 = nimg; k.bs1 = static_cast<long>(96) * M * 64;
    Epilogue e;
    e.out_f32 = u.scores; e.ldo = Mpad; e.obs0 = static_cast<long>(Ncap) * Mpad; e.obs1 = static_cast<long>(8) * Ncap * Mpad;
    e.alpha = 0.125f;  // == scaling q by 64^-0.5 before q k^T (exact: power of two)
    gemm(c, a, k, e);
  }
  softmax_rows(c, u.scores, Mpad, static_cast<long>(u.S) * 8, M, m->kpm + static_cast<long>(img0) * M, 8 * Ncap, M,
               nullptr, u.prob.hi, u.prob.lo, Mpad);
  {
    Operand a = act_op(u.prob.hi, u.prob.lo, Ncap, M, Mpad);
    a.nb0 = 8; a.bs0 = static_cast<long>(Ncap) * Mpad; a.nb1 = nimg; a.bs1 = static_cast<long>(8) * Ncap * Mpad;
    Operand v = act_op(m->vt_hi + voff, m->vt_lo + voff, 64, M, Mpad);
    v.nb0 = 8; v.bs0 = static_cast<long>(64) * Mpad; v.nb1 = nimg; v.bs1 = static_cast<long>(6144) * Mpad;
    Epilogue e;
    e.out_hi = u.o.hi; e.out_lo = u.o.lo; e.ldo = 512; e.obs0 = 64; e.obs1 = static_cast<long>(Ncap) * 512;
    gemm(c, a, v, e);
  }
}

// One decoder pass over the token at position *tpos of every sequence of decoders d0 .. d0 + b.nd - 1 (pre-norm layer,
// transformer.py:430-454, with self-attention K/V cached and the cross-attention K/V precomputed per image); decoder
// d0 + i reads its tokens at tokens[i] (row stride tstride[i]).  img0: first image of the batch slice the sequences
// belong to; nimg images x Ncap sequences each, per decoder.
void decoder_step(Ctx* c, OmniModel* m, int d0, StepBufs& b, const int* const tokens[], const int tstride[], int img0,
                  int nimg, bool want_logits) {
  DecodeBufs& u = b.all;
  const int nd = b.nd, d1 = d0 + nd - 1, S = u.S / nd;
  const bool two = nd == 2;
  embed_ln(c, tokens[0], tstride[0], u.tpos, u.S, m->word_emb, m->pos_emb[d0], m->emb_norm.g, m->emb_norm.b, u.x, u.qpos,
           two ? S : 0, two ? tokens[1] : nullptr, two ? tstride[1] : 0, two ? m->pos_emb[d1] : nullptr,
           two ? u.qpos + 512 : nullptr);
  const float* qpos = u.qpos;
  if (u.skinny) {
    // At most 32 live sequences (one per image, or up to 16 prompts per image in the pt loop): every linear is a skinny
    // fp32 GEMV (exact fp32 weights, one warp per output column), no operand splitting, no tensor-core tile padding.
    const int d = d0;
    auto lin = [&](const float* x, int K, const Lin& w, int act, float* out, const float* resid) {
      gemv_rows(c, x, nullptr, 1 << 30, K, w.wf, w.b, resid, w.w.N, out, w.w.N, S, w.w.N, K, act);
    };
    c->skip_scope = true;  // (timing experiments: alm_set_option debug_skip drops kernel classes inside the layers)
    if (c->fuse_ln_gemv && u.fused_xattn) {
      // same arithmetic, 13 fewer dependent launches per token: every pre-LayerNorm (+ query position) is applied by the
      // GEMV that consumes it, on its own staged copy of the rows
      auto lnlin = [&](const LNW& n, const float* pos, int pos_split, const float* W_, const float* b_, int N_, int act,
                       float* out, long ldo) {
        gemv_rows(c, u.x, nullptr, 1 << 30, 512, W_, b_, nullptr, 0, out, ldo, S, N_, 512, act, n.g, n.b, 1e-5f, pos, pos_split);
      };
      for (int l = 0; l < 4; ++l) {
        const DecLayerW& w = m->dec[d][l];
        lnlin(w.n1, qpos, 1024, w.sa_qkv_f, w.sa_qkv_b, 1536, ACT_NONE, u.qkv, 1536);   // q | k from LN(x)+pos, v from LN(x)
        self_attn_step(c, u.qkv, u.qkv + 1024, u.kc[l], u.vc[l], S, u.tpos, u.Tmax, nullptr, nullptr, u.attf, 1536, 1536,
                       u.anc);
        lin(u.attf, 512, w.sa_out, ACT_NONE, u.x, u.x);
        lnlin(w.n2, qpos, 1 << 30, w.ca_q.wf, w.ca_q.b, 512, ACT_NONE, u.qf, 512);
        cross_attn(c, m, u, d * 4 + l, img0, nimg, want_logits);
        lin(u.of, 512, w.ca_out, ACT_NONE, u.x, u.x);
        lnlin(w.n3, nullptr, 0, w.l1.wf, w.l1.b, 2048, ACT_RELU, u.hidf, 2048);
        lin(u.hidf, 2048, w.l2, ACT_NONE, u.x, u.x);
      }
      c->skip_scope = false;
      if (!want_logits) return;
      lnlin(m->dec_norm[d], nullptr, 0, m->head[d][0].wf, m->head[d][0].b, 512, ACT_RELU, u.h0f, 512);
      lin(u.h0f, 512, m->head[d][1], ACT_RELU, u.h1f, nullptr);
      lin(u.h1f, 512, m->head[d][2], ACT_NONE, u.logits, nullptr);
      return;
    }
    for (int l = 0; l < 4; ++l) {
      const DecLayerW& w = m->dec[d][l];
      gather_ln(c, u.x, 512, nullptr, 1, 512, S, w.n1.g, w.n1.b, 1e-5f, false, qpos, 0, u.lnf, 512, nullptr, nullptr, 512,
                nullptr, nullptr, u.lnpf);
      // q|k from LN(x)+pos and v from LN(x) in ONE launch: the fp32 in_proj rows are contiguous (q, k, v)
      gemv_rows(c, u.lnpf, u.lnf, 1024, 512, w.sa_qkv_f, w.sa_qkv_b, nullptr, 0, u.qkv, 1536, S, 1536, 512, ACT_NONE);
      self_attn_step(c, u.qkv, u.qkv + 1024, u.kc[l], u.vc[l], S, u.tpos, u.Tmax, nullptr, nullptr, u.attf, 1536, 1536,
                       u.anc);
      lin(u.attf, 512, w.sa_out, ACT_NONE, u.x, u.x);
      gather_ln(c, u.x, 512, nullptr, 1, 512, S, w.n2.g, w.n2.b, 1e-5f, false, qpos, 0, nullptr, 512, nullptr, nullptr, 512,
                nullptr, nullptr, u.lnpf);
      lin(u.lnpf, 512, w.ca_q, ACT_NONE, u.qf, nullptr);
      cross_attn(c, m, u, d * 4 + l, img0, nimg, want_logits);
      lin(u.of, 512, w.ca_out, ACT_NONE, u.x, u.x);
      gather_ln(c, u.x, 512, nullptr, 1, 512, S, w.n3.g, w.n3.b, 1e-5f, false, nullptr, 0, u.lnf, 512, nullptr, nullptr, 512,
                nullptr, nullptr);
      lin(u.lnf, 512, w.l1, ACT_RELU, u.hidf, nullptr);
      lin(u.hidf, 2048, w.l2, ACT_NONE, u.x, u.x);
    }
    c->skip_scope = false;
    if (!want_logits) return;
    gather_ln(c, u.x, 512, nullptr, 1, 512, S, m->dec_norm[d].g, m->dec_norm[d].b, 1e-5f, false, nullptr, 0, u.lnf, 512,
              nullptr, nullptr, 512, nullptr, nullptr);
    lin(u.lnf, 512, m->head[d][0], ACT_RELU, u.h0f, nullptr);
    lin(u.h0f, 512, m->head[d][1], ACT_RELU, u.h1f, nullptr);
    lin(u.h1f, 512, m->head[d][2], ACT_NONE, u.logits, nullptr);
    return;
  }
  // Tensor-core step.  Every LayerNorm is one launch over all rows and every linear one GEMM; with nd 2 rows [S, 2S)
  // take decoder d1's affine, query position and weights (linear2: a batch of two over the load_lin_pair slab), so each
  // row's arithmetic is the single-decoder step's.
  auto ln = [&](const LNW& n0, const LNW& n1, bool pos, const SplitBuf& out, const SplitBuf& out_pos) {
    gather_ln(c, u.x, 512, nullptr, 1, 512, u.S, n0.g, n0.b, 1e-5f, false, pos ? qpos : nullptr, 0, nullptr, 0, out.hi,
              out.lo, 512, out_pos.hi, out_pos.lo, nullptr, two ? S : 0, two ? n1.g : nullptr, two ? n1.b : nullptr,
              two && pos ? qpos + 512 : nullptr);
  };
  auto lin = [&](const SplitBuf& a, const Lin& l0, const Lin& l1, int act, float* out_f32, SplitBuf* out_split,
                 bool resid) {
    if (two) linear2(c, a, S, l0, l1, act, out_f32, out_split, resid ? u.x : nullptr);
    else linear(c, a, S, l0, act, out_f32, out_split, resid ? u.x : nullptr);
  };
  // the self-attention step runs over all rows at once when each decoder's rows alone would take the same kernel
  auto wide = [&](long rows) { return c->sattn_wide && rows * 8 <= 4L * c->num_sms; };
  const bool one_sattn = wide(S) == wide(u.S);
  c->skip_scope = true;
  for (int l = 0; l < 4; ++l) {
    const DecLayerW& w = m->dec[d0][l];
    const DecLayerW& w1 = m->dec[d1][l];
    // --- self attention
    ln(w.n1, w1.n1, true, u.ln, u.lnp);
    lin(u.lnp, w.sa_qk, w1.sa_qk, ACT_NONE, u.qk, nullptr, false);
    lin(u.ln, w.sa_v, w1.sa_v, ACT_NONE, u.v, nullptr, false);
    for (int i = 0; i < (one_sattn ? 1 : nd); ++i) {
      DecodeBufs& v = one_sattn ? u : b.v(i);
      self_attn_step(c, v.qk, v.v, v.kc[l], v.vc[l], v.S, v.tpos, v.Tmax, v.att.hi, v.att.lo, nullptr, 1024, 512, v.anc);
    }
    lin(u.att, w.sa_out, w1.sa_out, ACT_NONE, u.x, nullptr, true);
    // --- cross attention, each decoder against its own layer of the per-image cached K / V^T
    ln(w.n2, w1.n2, true, SplitBuf{}, u.lnp);
    if (u.Ncap == 1) lin(u.lnp, w.ca_q, w1.ca_q, ACT_NONE, u.qf, nullptr, false);
    else lin(u.lnp, w.ca_q, w1.ca_q, ACT_NONE, nullptr, &u.q, false);
    for (int i = 0; i < nd; ++i) cross_attn(c, m, b.v(i), (d0 + i) * 4 + l, img0, nimg, want_logits);
    lin(u.o, w.ca_out, w1.ca_out, ACT_NONE, u.x, nullptr, true);
    // --- FFN
    ln(w.n3, w1.n3, false, u.ln, SplitBuf{});
    lin(u.ln, w.l1, w1.l1, ACT_RELU, nullptr, &u.hid, false);
    lin(u.hid, w.l2, w1.l2, ACT_NONE, u.x, nullptr, true);
  }
  c->skip_scope = false;
  if (!want_logits) return;
  ln(m->dec_norm[d0], m->dec_norm[d1], false, u.ln, SplitBuf{});
  lin(u.ln, m->head[d0][0], m->head[d1][0], ACT_RELU, nullptr, &u.h0, false);
  lin(u.h0, m->head[d0][1], m->head[d1][1], ACT_RELU, nullptr, &u.h1, false);
  lin(u.h1, m->head[d0][2], m->head[d1][2], ACT_NONE, u.logits, nullptr, false);
}

// Sleep (do not spin) until everything enqueued on `s` has finished.  The decode loops wait for the GPU several
// times per batch and a serving process keeps several contexts (host threads) per GPU in flight: spinning threads
// would fight over the host cores (cgroup quotas are far below the visible CPU count on the GPU boxes).  The
// device-to-pageable-host copies that follow each wait would otherwise spin inside cudaMemcpyAsync.
void wait_stream(Ctx* c, cudaStream_t s) {
  if (!c->ev_block)
    ALM_CHECK_CUDA(cudaEventCreateWithFlags(&c->ev_block, cudaEventBlockingSync | cudaEventDisableTiming));
  ALM_CHECK_CUDA(cudaEventRecord(c->ev_block, s));
  ALM_CHECK_CUDA(cudaEventSynchronize(c->ev_block));
}

// The context's character sets (alm_omni_set_rec_charset) against one decode, before any device work: the sets must
// cover the checkpoint's characters, and row sets are read by alm_omni_decode_at alone, one per row of its B x cap
// (at_rows; -1 for every other entry).
void check_rec_charset(const Ctx* c, const alm_decode_cfg& cfg, long at_rows) {
  if (c->rec_cs_sets == 0) return;
  const std::string fn = "alm_omni_set_rec_charset: ";
  ALM_REQUIRE(c->rec_cs_chars == cfg.recog_pad - cfg.num_bins - 1, ALM_ERR_INVALID,
              fn + "n_chars must be recog_pad - num_bins - 1 = " + std::to_string(cfg.recog_pad - cfg.num_bins - 1) +
                  ", the checkpoint's characters");
  for (int k = 0; k < c->rec_cs_sets; ++k) {
    const uint8_t* a = c->rec_cs_allowed.data() + static_cast<size_t>(k) * c->rec_cs_chars;
    ALM_REQUIRE(std::any_of(a, a + c->rec_cs_chars, [](uint8_t v) { return v != 0; }), ALM_ERR_INVALID,
                fn + "set " + std::to_string(k) + " is empty");
  }
  if (c->rec_cs_rows.empty()) return;
  ALM_REQUIRE(at_rows >= 0, ALM_ERR_INVALID, fn + "row sets are read by alm_omni_decode_at only (set them again with "
                                                  "row_set NULL for the other decodes)");
  ALM_REQUIRE(static_cast<long>(c->rec_cs_rows.size()) == at_rows, ALM_ERR_INVALID,
              fn + "n_rows must be B x cap = " + std::to_string(at_rows) + " of this alm_omni_decode_at");
  for (int32_t k : c->rec_cs_rows)
    ALM_REQUIRE(k >= 0 && k < c->rec_cs_sets, ALM_ERR_INVALID, fn + "a row's set index is outside [0, n_sets)");
}

struct HeadArgs {
  bool on = false;
  HeadCfg cfg{};
  int* tokens = nullptr;
  int tstride = 0, n_prompt_m1 = 0;
  float* probs = nullptr;
  int pstride = 0;
  int* finished = nullptr;
  int* ntok = nullptr;
  int seqs_per_image = 1;
  int nsoft = 0;  // logits entering the softmax (V, or V - vie_categories for the KIE poly/rec loops)
  int topk = 0;   // rec loop: > 0 = also record the k best classes per step at cand_ids / cand_probs [seq][step][k]
  int* cand_ids = nullptr;
  float* cand_probs = nullptr;
  int beams = 0;  // rec loop: > 0 = beam search of this width over groups of `beams` adjacent sequences (beam_select)
  float* bscore = nullptr;
  int* blen = nullptr;
  int* anc = nullptr;
};

// The token choice of one step of decoder d from u.logits: beam search, top-k candidates or greedy (none when !h.on).
void select_heads(Ctx* c, OmniModel* m, int d, DecodeBufs& u, const HeadArgs& h) {
  if (h.on && h.beams > 0)
    beam_select(c, u.logits, u.S / h.beams, h.beams, m->V, h.nsoft ? h.nsoft : m->V, h.cfg, h.tokens, h.tstride, u.tpos,
                h.n_prompt_m1, h.probs, h.pstride, h.bscore, h.blen, h.anc, u.Tmax);
  else if (h.on && h.topk > 0)
    head_select_topk(c, u.logits, u.S, m->V, h.nsoft ? h.nsoft : m->V, h.cfg, h.tokens, h.tstride, u.tpos, h.n_prompt_m1,
                     h.probs, h.pstride, h.topk, h.cand_ids, h.cand_probs, h.pstride * h.topk);
  else if (h.on)
    head_select(c, u.logits, u.S, m->V, h.nsoft ? h.nsoft : m->V, d, h.cfg, h.tokens, h.tstride, u.tpos, h.n_prompt_m1, h.probs, h.pstride,
                h.finished, h.ntok, h.seqs_per_image);
}

// What a captured step of decoder d over `u` depends on: shapes, pointers and every option its launches read.
std::vector<long> step_key(Ctx* c, OmniModel* m, int d, DecodeBufs& u, const int* tokens, int tstride, int img0, int nimg,
                           const HeadArgs& h) {
  return {d, u.S, u.Ncap, u.Tmax, img0, nimg, m->M, h.on ? 1 : 0, c->nsplit,
                           reinterpret_cast<long>(u.x), reinterpret_cast<long>(tokens), tstride,
                           reinterpret_cast<long>(h.probs), reinterpret_cast<long>(h.finished), h.n_prompt_m1,
                           reinterpret_cast<long>(m->kc_hi), reinterpret_cast<long>(u.kc[3]), h.cfg.pt_eos, h.cfg.num_bins,
                           h.cfg.rec_eos, h.cfg.recog_pad, reinterpret_cast<long>(c->trace_buf), h.nsoft, h.cfg.vie, c->xattn_impl, c->gemm_grid_cap, c->small_grid_cap, c->debug_skip, c->xattn_ctas_per_sm, c->sattn_wide, c->xattn_wg, c->fuse_ln_gemv,
                           reinterpret_cast<long>(m->key_len), u.mq_grid, u.mq_parts, h.topk,
                           reinterpret_cast<long>(h.cand_ids), reinterpret_cast<long>(h.cand_probs), h.beams,
                           reinterpret_cast<long>(h.bscore), reinterpret_cast<long>(u.anc), reinterpret_cast<long>(u.loc),
                           reinterpret_cast<long>(h.cfg.cs_allowed), reinterpret_cast<long>(h.cfg.cs_set)};
}

// n replays of one step `body`.  The step (all ~62 launches + the counter increment) is captured once into a CUDA
// graph per distinct `key` (shape, pointer) signature and replayed: the per-token host cost drops from ~62 launches
// to one cudaGraphLaunch.  Graphs off: the body runs as it is.
template <class Body>
void run_graph(Ctx* c, OmniModel* m, const std::vector<long>& key, int n, const Body& body) {
  if (!c->use_graphs || c->profile_gemm || c->gemm_impl != 0) {
    for (int i = 0; i < n; ++i) body();
    return;
  }
  auto it = m->step_graphs.find(key);
  if (it == m->step_graphs.end()) {
    if (m->step_graphs.size() > 64) {
      for (auto& kv : m->step_graphs) cudaGraphExecDestroy(kv.second.exec);
      m->step_graphs.clear();
    }
    const long before = c->launches;
    cudaGraph_t graph = nullptr;
    ALM_CHECK_CUDA(cudaStreamBeginCapture(c->stream, cudaStreamCaptureModeThreadLocal));
    try {
      body();
    } catch (...) {
      cudaStreamEndCapture(c->stream, &graph);
      if (graph) cudaGraphDestroy(graph);
      throw;
    }
    ALM_CHECK_CUDA(cudaStreamEndCapture(c->stream, &graph));
    OmniModel::StepGraph sg{nullptr, c->launches - before};
    c->launches = before;
    cudaError_t e = cudaGraphInstantiate(&sg.exec, graph, 0);
    cudaGraphDestroy(graph);
    if (e != cudaSuccess) throw AlmError{ALM_ERR_CUDA, std::string("cudaGraphInstantiate: ") + cudaGetErrorString(e)};
    it = m->step_graphs.emplace(key, sg).first;
  }
  for (int i = 0; i < n; ++i) ALM_CHECK_CUDA(cudaGraphLaunch(it->second.exec, c->stream));
  c->launches += it->second.launches * n;
}

// `n` consecutive token steps of decoders d0 .. d0 + b.nd - 1: their layers, then each decoder's head selection, then
// the shared position counter.  One graph key per decoder, joined by -1 (no single-decoder key has that length).
void run_steps(Ctx* c, OmniModel* m, int d0, StepBufs& b, const int* const tokens[], const int tstride[], int img0,
               int nimg, int n, const HeadArgs h[]) {
  if (n <= 0) return;
  ALM_REQUIRE(h[0].on == h[b.nd - 1].on, ALM_ERR_STATE, "joint decoder step: both halves select or neither");
  std::vector<long> key;
  for (int i = 0; i < b.nd; ++i) {
    const std::vector<long> k = step_key(c, m, d0 + i, b.v(i), tokens[i], tstride[i], img0, nimg, h[i]);
    if (i > 0) key.push_back(-1);
    key.insert(key.end(), k.begin(), k.end());
  }
  run_graph(c, m, key, n, [&] {
    decoder_step(c, m, d0, b, tokens, tstride, img0, nimg, h[0].on);
    for (int i = 0; i < b.nd; ++i) select_heads(c, m, d0 + i, b.v(i), h[i]);
    add_i32(c, b.all.tpos, 1);
  });
}

// The joint pass serves the tensor-core step of the fused cross-attention over one row per instance; the fp32 GEMV
// step (<= 32 single-instance sequences), the unfused cross-attention and beam search keep the single-decoder steps,
// and so does every decode with the "joint_decode" option off.
bool joint_pass_ok(Ctx* c, int B, int Ncap, bool beams) {
  const bool skinny = B * Ncap <= 32 && Ncap == 1;
  return c->joint_decode && !skinny && !beams && (c->xattn_impl == 0 || c->xattn_impl == 2);
}

// The point loop (transformer.py:102-141) of images img0 .. img0 + nimg - 1 with P prompts each: sequence
// (b - img0) P + p of pt_tok [S][n_prompt + pt_steps], prompt tokens first, EOS per sequence in finished / ntok
// (zeroed by the caller).  Runs in chunks of 16 steps with one small sync after each to stop once every sequence chose
// pt_eos; after the last chunk only when check_last.  Returns whether every sequence had chosen pt_eos at the last check.
bool pt_loop(Ctx* c, OmniModel* m, const HeadCfg& hc, int img0, int nimg, int P, int n_prompt, int pt_steps,
             bool check_last, int* pt_tok, float* pt_prob, int* finished, int* ntok) {
  const int S = nimg * P, Tpt = n_prompt + pt_steps;
  StepBufs u = alloc_decode(c, m, 1, nimg, P, Tpt - 1, true, img0);
  fill_i32(c, u.all.tpos, 1, 0);
  const int* const tok[1] = {pt_tok};
  HeadArgs off;
  run_steps(c, m, 0, u, tok, &Tpt, img0, nimg, n_prompt - 1, &off);  // prompt tokens only fill the caches
  HeadArgs h;
  h.on = true; h.cfg = hc; h.tokens = pt_tok; h.tstride = Tpt; h.n_prompt_m1 = n_prompt - 1;
  h.probs = pt_prob; h.pstride = pt_steps;
  h.finished = finished; h.ntok = ntok; h.seqs_per_image = 1;  // EOS per sequence, also with several prompts per image
  std::vector<int> fin(S);
  bool all_done = false;
  for (int done = 0; done < pt_steps && !all_done;) {
    const int chunk = std::min(16, pt_steps - done);
    run_steps(c, m, 0, u, tok, &Tpt, img0, nimg, chunk, &h);
    done += chunk;
    if (done < pt_steps || check_last) {  // every sequence hit EOS?  (one small sync per 16 tokens)
      wait_stream(c, c->stream);
      ALM_CHECK_CUDA(cudaMemcpyAsync(fin.data(), finished, S * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
      ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
      all_done = std::all_of(fin.begin(), fin.end(), [](int v) { return v != 0; });
    }
  }
  return all_done;
}

// The settings of every decode loop: the decoder's GEMM grid cap and, with alm_omni_set_decode_priority, the loops on
// internal high-priority streams (fork from / join to the caller's stream); undone when the scope ends.
struct DecodeScope {
  Ctx* c;
  cudaStream_t user;
  bool swapped = false;
  explicit DecodeScope(Ctx* c_) : c(c_), user(c_->stream) {
    if (c->decode_priority) {
      int least = 0, greatest = 0;
      ALM_CHECK_CUDA(cudaDeviceGetStreamPriorityRange(&least, &greatest));
      if (!c->stream_hi) {
        ALM_CHECK_CUDA(cudaStreamCreateWithPriority(&c->stream_hi, cudaStreamNonBlocking, greatest));
        ALM_CHECK_CUDA(cudaEventCreateWithFlags(&c->ev_prio, cudaEventDisableTiming));
      }
      if (!c->stream2) ALM_CHECK_CUDA(cudaStreamCreateWithPriority(&c->stream2, cudaStreamNonBlocking, greatest));
      ALM_CHECK_CUDA(cudaEventRecord(c->ev_prio, c->stream));
      ALM_CHECK_CUDA(cudaStreamWaitEvent(c->stream_hi, c->ev_prio, 0));
      c->stream = c->stream_hi;
      swapped = true;
    }
    c->gemm_grid_cap = c->dec_grid_cap;
  }
  ~DecodeScope() {
    c->gemm_grid_cap = 0;
    if (swapped) {
      cudaStream_t hi = c->stream;
      c->stream = user;
      if (cudaEventRecord(c->ev_prio, hi) == cudaSuccess) cudaStreamWaitEvent(user, c->ev_prio, 0);
    }
  }
};

// level 0 of alm_omni_decode_dense: per sequence whether it saturated; when one did, its tokens [S][Tpt] and counts
struct Level0 {
  bool saturated = false;
  std::vector<uint8_t> sat;
  std::vector<int> ntok, tok;
};

// What poly_rec returns on the host, per row r (page-major, Ncap rows per page): tok[d] [r][3 + length] ([x, y, sos] +
// generated) and prob[d] [r][length] of the polygon (d 1) and the recognition loop (d 2; with beams none, their
// hypothesis 0 is the reading), candidates [r][rec_length][K], n-best lists ids / probs [r][W][rec_length] and scores
// [r][W], locations [r][rec_length][5]; each list empty unless its option is on.
struct PolyRec {
  std::vector<int> tok[3], cand_ids, beam_ids;
  std::vector<float> prob[3], cand_probs, beam_probs, beam_scores, loc;
};

// Polygon and recognition loops (transformer.py:249-284 ; :153-185 for KIE) of pages img0 .. img0 + pts.size() - 1,
// Ncap rows per page: row n of page img0 + i is [x, y, sos] of pts[i][n], a dead row 0, 0, sos past pts[i]'s end.  The
// context's rec_topk / rec_beams / rec_locations add candidates, beam search or locations to the recognition loop, and
// its character sets (rec_cs_sets > 0) restrict the recognition loop's choice: row n of page img0 + i reads with set
// row_set[(img0 + i) * row_stride + n] (row_set null, and dead rows: set 0).
// The two loops only depend on the points, not on each other.  With one row per instance they run as one joint pass
// while both have steps left, then the longer loop finishes alone; otherwise (beams, the fp32 GEMV step, the unfused
// cross-attention) they run concurrently on two streams.  `done` (if any) is recorded on the caller's stream once every
// loop is enqueued.
PolyRec poly_rec(Ctx* c, const alm_decode_cfg& cfg, const HeadCfg& hc, int img0, const std::vector<Points>& pts, int Ncap,
                 cudaEvent_t done, const int32_t* row_set = nullptr, int row_stride = 0) {
  OmniModel* m = c->omni;
  Arena& ws = c->ws;
  const int nimg = static_cast<int>(pts.size()), Si = nimg * Ncap;  // poly / rec instances
  const int K = c->rec_topk, Wb = c->rec_beams;
  const bool Lc = c->rec_locations;
  const int lens[3] = {0, cfg.poly_length, cfg.rec_length};
  if (!c->stream2) ALM_CHECK_CUDA(cudaStreamCreateWithFlags(&c->stream2, cudaStreamNonBlocking));
  if (!c->ev_fork) {
    ALM_CHECK_CUDA(cudaEventCreateWithFlags(&c->ev_fork, cudaEventDisableTiming));
    ALM_CHECK_CUDA(cudaEventCreateWithFlags(&c->ev_join, cudaEventDisableTiming));
  }
  cudaStream_t s0 = c->stream, s1 = c->decode_streams == 2 ? c->stream2 : c->stream;
  // sequences per instance: the rec loop with beams runs the W hypotheses of an instance as adjacent rows of its image
  const int rows_per[3] = {1, 1, Wb > 0 ? Wb : 1};
  int* toks[3] = {nullptr, nullptr, nullptr};
  float* prbs[3] = {nullptr, nullptr, nullptr};
  std::vector<int> h_prompt[3];
  for (int phase = 1; phase <= 2; ++phase) {  // [x, y, sos] per instance (transformer.py:252,268 ; :153,172); dead rows 0,0,sos
    const int T = 3 + lens[phase], R = rows_per[phase];
    h_prompt[phase].assign(static_cast<size_t>(Si) * R * T, 0);
    for (int b = 0; b < nimg; ++b)
      for (int n = 0; n < Ncap; ++n)
        for (int w = 0; w < R; ++w) {
          int* row = &h_prompt[phase][((static_cast<size_t>(b) * Ncap + n) * R + w) * T];
          if (n < static_cast<int>(pts[b].size())) {
            row[0] = pts[b][n].first; row[1] = pts[b][n].second;
          }
          row[2] = phase == 1 ? cfg.poly_sos : cfg.rec_sos;
        }
    toks[phase] = ws.get<int>(static_cast<size_t>(Si) * R * T);
    prbs[phase] = ws.get<float>(static_cast<size_t>(Si) * R * (T - 3));
    ALM_CHECK_CUDA(cudaMemcpyAsync(toks[phase], h_prompt[phase].data(), h_prompt[phase].size() * sizeof(int),
                                   cudaMemcpyHostToDevice, s0));
  }
  // the caller's character sets (alm_omni_set_rec_charset) for the recognition loop's head selection alone: the sets,
  // and each instance's set when rows differ; nothing is allocated or copied without them
  HeadCfg rc = hc;
  std::vector<int> h_cs;
  if (c->rec_cs_sets > 0) {
    uint8_t* d_allowed = ws.get<uint8_t>(c->rec_cs_allowed.size());
    ALM_CHECK_CUDA(cudaMemcpyAsync(d_allowed, c->rec_cs_allowed.data(), c->rec_cs_allowed.size(), cudaMemcpyHostToDevice,
                                   s0));
    rc.cs_allowed = d_allowed;
    if (row_set) {
      h_cs.assign(Si, 0);
      for (int b = 0; b < nimg; ++b)
        for (size_t n = 0; n < pts[b].size(); ++n)
          h_cs[static_cast<size_t>(b) * Ncap + n] = row_set[static_cast<size_t>(img0 + b) * row_stride + n];
      int* d_cs = ws.get<int>(Si);
      ALM_CHECK_CUDA(cudaMemcpyAsync(d_cs, h_cs.data(), h_cs.size() * sizeof(int), cudaMemcpyHostToDevice, s0));
      rc.cs_set = d_cs;
    }
  }
  // rec candidates on the device: [Si sequences][rec_length][K], every entry written by the rec loop
  const size_t cand_n = static_cast<size_t>(Si) * cfg.rec_length * K;
  int* d_cand_ids = K > 0 ? ws.get<int>(cand_n) : nullptr;
  float* d_cand_probs = K > 0 ? ws.get<float>(cand_n) : nullptr;
  // beam state [Si * W] (score, length), ancestry [Si * W][rec Tmax], n-best lists [Si][W][rec_length] and [Si][W]
  const size_t nb = static_cast<size_t>(Si) * Wb, bl_n = nb * cfg.rec_length;
  float* d_bscore = Wb > 0 ? ws.get<float>(nb) : nullptr;
  int* d_blen = Wb > 0 ? ws.get<int>(nb) : nullptr;
  int* d_anc = Wb > 0 ? ws.get<int>(nb * (2 + cfg.rec_length)) : nullptr;
  int* d_bids = Wb > 0 ? ws.get<int>(bl_n) : nullptr;
  float* d_bprobs = Wb > 0 ? ws.get<float>(bl_n) : nullptr;
  float* d_bscores = Wb > 0 ? ws.get<float>(nb) : nullptr;
  // character locations on the device: [Si sequences][rec_length][5], every entry written by the rec loop
  const size_t loc_n = Lc ? static_cast<size_t>(Si) * cfg.rec_length * 5 : 0;
  float* d_loc = Lc ? ws.get<float>(loc_n) : nullptr;
  auto heads = [&](int phase) {  // head selection of the polygon (1) or recognition (2) loop
    HeadArgs h;
    h.on = true; h.cfg = phase == 2 ? rc : hc; h.tokens = toks[phase]; h.tstride = 3 + lens[phase]; h.n_prompt_m1 = 2;
    h.probs = prbs[phase]; h.pstride = lens[phase]; h.seqs_per_image = Ncap;
    h.nsoft = m->V - m->vie;  // logits[:, -1, :-vie_categories] (transformer.py:156,176)
    if (phase == 2 && K > 0) { h.topk = K; h.cand_ids = d_cand_ids; h.cand_probs = d_cand_probs; }
    if (phase == 2 && Wb > 0) { h.beams = Wb; h.bscore = d_bscore; h.blen = d_blen; h.anc = d_anc; }
    return h;
  };
  auto locations = [&](DecodeBufs& u) {  // the rec loop's character locations
    size_t pf = 0;
    int groups = 0;
    rec_locate_plan(c, nimg, Ncap, m->M, m->mixed ? m->page_keys.data() + img0 : nullptr, &u.loc_ks, &pf, &groups);
    u.loc = d_loc;
    u.loc_L = lens[2];
    u.loc_partial = ws.get<float>(pf);
    u.loc_counters = ws.get<int>(groups);
    // a memset, not a kernel: locations add exactly one launch per generated rec step
    ALM_CHECK_CUDA(cudaMemsetAsync(u.loc_counters, 0, groups * sizeof(int), c->stream));
  };
  if (joint_pass_ok(c, nimg, Ncap, Wb > 0)) {
    StepBufs jb = alloc_decode(c, m, 2, nimg, Ncap, 2 + std::max(lens[1], lens[2]), false, img0);
    fill_i32(c, jb.all.tpos, 1, 0);
    if (Lc) locations(jb.half[1]);
    const int* const jt[2] = {toks[1], toks[2]};
    const int js[2] = {3 + lens[1], 3 + lens[2]};
    const HeadArgs off[2], hs[2] = {heads(1), heads(2)};
    run_steps(c, m, 1, jb, jt, js, img0, nimg, 2, off);  // the prompts [x, y, sos] only fill the caches
    const int both = std::min(lens[1], lens[2]);
    run_steps(c, m, 1, jb, jt, js, img0, nimg, both, hs);
    for (int i = 0; i < 2; ++i) {  // the longer loop alone
      StepBufs alone{1, jb.half[i]};
      run_steps(c, m, 1 + i, alone, &jt[i], &js[i], img0, nimg, lens[1 + i] - both, &hs[i]);
    }
  } else {
    ALM_CHECK_CUDA(cudaEventRecord(c->ev_fork, s0));
    ALM_CHECK_CUDA(cudaStreamWaitEvent(s1, c->ev_fork, 0));
    try {
      for (int phase = 1; phase <= 2; ++phase) {
        c->stream = (phase == 1) ? s0 : s1;
        const int len = lens[phase], T = 3 + len;
        const bool beams = phase == 2 && Wb > 0;
        StepBufs u = alloc_decode(c, m, 1, nimg, Ncap * rows_per[phase], T - 1, false, img0);
        fill_i32(c, u.all.tpos, 1, 0);
        if (beams) {  // the prompt [x, y, sos] is cached in every beam's own row
          anc_identity(c, d_anc, static_cast<int>(nb), T - 1);
          u.all.anc = d_anc;
        }
        if (phase == 2 && Lc) locations(u.all);
        const HeadArgs off, h = heads(phase);
        run_steps(c, m, phase, u, &toks[phase], &T, img0, nimg, 2, &off);
        run_steps(c, m, phase, u, &toks[phase], &T, img0, nimg, len, &h);
        if (beams)
          beam_backtrace(c, toks[phase], T, prbs[phase], len, d_bscore, d_blen, d_anc, T - 1, Si, Wb, len, 3, c->beam_alpha,
                         d_bids, d_bprobs, d_bscores);
      }
    } catch (...) {
      c->stream = s0;
      cudaStreamSynchronize(s1);
      throw;
    }
    c->stream = s0;
    ALM_CHECK_CUDA(cudaEventRecord(c->ev_join, s1));
    ALM_CHECK_CUDA(cudaStreamWaitEvent(s0, c->ev_join, 0));
  }
  if (done) ALM_CHECK_CUDA(cudaEventRecord(done, s0));
  wait_stream(c, s0);
  PolyRec r;
  auto fetch = [&](auto& host, const auto* dev, size_t n) {
    host.resize(n);
    ALM_CHECK_CUDA(cudaMemcpyAsync(host.data(), dev, n * sizeof(*dev), cudaMemcpyDeviceToHost, s0));
  };
  for (int phase = 1; phase <= 2; ++phase)
    if (phase == 1 || Wb == 0) {  // beams: only the n-best lists leave the device
      fetch(r.tok[phase], toks[phase], static_cast<size_t>(Si) * (3 + lens[phase]));
      fetch(r.prob[phase], prbs[phase], static_cast<size_t>(Si) * lens[phase]);
    }
  if (K > 0) {
    fetch(r.cand_ids, d_cand_ids, cand_n);
    fetch(r.cand_probs, d_cand_probs, cand_n);
  }
  if (Wb > 0) {
    fetch(r.beam_ids, d_bids, bl_n);
    fetch(r.beam_probs, d_bprobs, bl_n);
    fetch(r.beam_scores, d_bscores, nb);
  }
  if (Lc) fetch(r.loc, d_loc, loc_n);
  ALM_CHECK_CUDA(cudaStreamSynchronize(s0));
  return r;
}

// The polygon and recognition stage of alm_omni_decode, _prompts, _kie and _at at given points.  uniq[b] lists the
// (x, y) bins of image b, one row per entry (Ncap = the longest list); instance n of slot q (image q / P) takes the
// result of entry slot_inst[q][n] of its image.  Writes poly / rec / rec_prob in alm_omni_decode's layout with maxI
// rows per slot, and keeps the candidate / beam / location lists of the context's settings in the model.
void poly_rec_loops(Ctx* c, const alm_decode_cfg& cfg, const HeadCfg& hc, int P, int maxI, const std::vector<Points>& uniq,
                    const std::vector<std::vector<int>>& slot_inst, int64_t* poly, int64_t* rec, float* rec_prob,
                    const int32_t* row_set = nullptr, int row_stride = 0) {
  OmniModel* m = c->omni;
  const int S = static_cast<int>(slot_inst.size()), K = c->rec_topk, Wb = c->rec_beams;
  const size_t L = cfg.rec_length, rows = static_cast<size_t>(S) * maxI;
  int Ncap = 0;
  for (const auto& u : uniq) Ncap = std::max(Ncap, static_cast<int>(u.size()));
  OmniModel::RecLists lists;  // [slot][max_inst][...]; instances past n_inst stay 0
  if (K > 0) {
    lists.cand_ids.assign(rows * L * K, 0);
    lists.cand_probs.assign(rows * L * K, 0.f);
  }
  if (Wb > 0) {
    lists.beam_ids.assign(rows * Wb * L, 0);
    lists.beam_probs.assign(rows * Wb * L, 0.f);
    lists.beam_scores.assign(rows * Wb, 0.f);
  }
  if (c->rec_locations) lists.rec_loc.assign(rows * L * 5, 0.f);
  if (Ncap > 0) {
    const PolyRec r = poly_rec(c, cfg, hc, 0, uniq, Ncap, c->ev_t[4], row_set, row_stride);
    c->timing_valid[1] = true;
    const size_t T1 = 3 + cfg.poly_length, T2 = 3 + L;
    for (int q = 0; q < S; ++q)
      for (int n = 0; n < static_cast<int>(slot_inst[q].size()); ++n) {
        // a deduplicated (x, y) carries its results to every slot holding it: entries [from, from + len) of row sq of
        // `src` to row o = (q, n) of `dst`
        const size_t sq = static_cast<size_t>(q / P) * Ncap + slot_inst[q][n], o = static_cast<size_t>(q) * maxI + n;
        auto carry = [&](const auto& src, size_t from, size_t len, auto* dst) {
          std::copy(src.begin() + from, src.begin() + from + len, dst + o * len);
        };
        carry(r.tok[1], sq * T1 + 3, cfg.poly_length, poly);
        if (Wb > 0) {  // hypothesis 0 is rec / rec_prob
          carry(r.beam_ids, sq * Wb * L, L, rec);
          carry(r.beam_probs, sq * Wb * L, L, rec_prob);
          carry(r.beam_ids, sq * Wb * L, Wb * L, lists.beam_ids.data());
          carry(r.beam_probs, sq * Wb * L, Wb * L, lists.beam_probs.data());
          carry(r.beam_scores, sq * Wb, Wb, lists.beam_scores.data());
        } else {
          carry(r.tok[2], sq * T2 + 3, L, rec);
          carry(r.prob[2], sq * L, L, rec_prob);
        }
        if (K > 0) {
          carry(r.cand_ids, sq * L * K, L * K, lists.cand_ids.data());
          carry(r.cand_probs, sq * L * K, L * K, lists.cand_probs.data());
        }
        if (!r.loc.empty()) carry(r.loc, sq * L * 5, L * 5, lists.rec_loc.data());
      }
    c->ws.release(m->ws_mark);
  }
  m->rec_lists = std::move(lists);
}

}  // namespace

// Greedy decoding of every encoded image.  Text spotting (transformer.py:234-286) and KIE (:143-217) share the
// pt loop and the batched poly / rec loops; they differ in the pt step pattern (x, y[, class]), in which decoded
// tokens form (x, y) instances and in the number of logits entering the poly / rec softmax.
// P prompts per image: token i of prompt p of image b is prompts[b * page_stride + p * n_prompt + i] (page_stride 0:
// one prompt set for every image).  The pt loop runs the B * P (image, prompt) slots as sequences b * P + p; every
// per-image output below is per slot, so with P == 1 a slot is an image.
// level0 (alm_omni_decode_dense's first reading, P = 1): a saturated sequence is reported in *level0 instead of failing
// the call, and when one is, the decode stops after the point loop with the tokens in *level0 and no output written.
void omni_decode_impl(Ctx* c, const int64_t* prompts, long page_stride, int P, int n_prompt, const alm_decode_cfg& cfg,
                      bool kie, int32_t* n_tok_out, int64_t* pt_tok_out, float* pt_prob_out, int32_t* n_inst,
                      int32_t* inst_pos, int64_t* pt, int64_t* poly, int64_t* rec, float* rec_prob,
                      bool points_only = false, Level0* level0 = nullptr) {
  OmniModel* m = c->omni;
  ALM_REQUIRE(m && m->encoded, ALM_ERR_STATE, "alm_omni_decode before alm_omni_encode");
  ALM_REQUIRE(c->xattn_impl != 1 || m->vt_hi, ALM_ERR_STATE, "xattn_impl 1 must be set before alm_omni_encode");
  ALM_REQUIRE(n_prompt >= 1 && n_prompt <= 16, ALM_ERR_INVALID, "pt prompt length");
  ALM_REQUIRE(cfg.pt_seq_length >= 1, ALM_ERR_INVALID, "pt_seq_length");
  // The reference default is --pt_seq_length 1024 (utils/parser.py:21) with a 5- or 7-token prompt: more steps than the
  // 1024-row position table (transformer.py:475) can serve.  It works because EOS ends the loop (:126) long before
  // step 1025 - n_prompt, where the embedding lookup (:312) would raise.  Same here: the loop is sized by the table,
  // and an image that is still alive when the table is exhausted is an error, as in the reference.
  const int pt_steps = std::min(cfg.pt_seq_length, 1025 - n_prompt);
  const bool pt_clamped = pt_steps < cfg.pt_seq_length;
  ALM_REQUIRE(cfg.vie_categories == m->vie, ALM_ERR_INVALID, "vie_categories does not match the loaded checkpoint");
  ALM_REQUIRE(kie == (m->vie > 0), ALM_ERR_INVALID, "use alm_omni_decode for text spotting and alm_omni_decode_kie for KIE");
  ALM_REQUIRE(m->kv_decoders == 3 || points_only, ALM_ERR_STATE,
              "the batch was encoded with kv_decoders < 3: only alm_omni_decode_points can run on it");
  ALM_REQUIRE(points_only || cfg.max_instances >= (pt_steps / 2), ALM_ERR_INVALID, "max_instances < pt_seq_length / 2");
  ALM_REQUIRE(points_only || cfg.poly_length == 32, ALM_ERR_UNSUPPORTED, "polygon length is fixed at 32 (transformer.py:254)");
  if (!points_only) check_rec_charset(c, cfg, -1);
  const int B = m->B;
  Arena& ws = c->ws;
  ws.release(m->ws_mark);
  HeadCfg hc{cfg.num_bins, cfg.pt_eos, cfg.rec_eos, cfg.recog_pad, m->vie};
  // recognition candidates per rec step (alm_omni_set_rec_candidates); they describe this decode or none
  const int K = points_only ? 0 : c->rec_topk;
  // beam width of the rec loop (alm_omni_set_rec_beams); the n-best lists describe this decode or none
  const int Wb = points_only ? 0 : c->rec_beams;
  ALM_REQUIRE(K == 0 || Wb == 0, ALM_ERR_INVALID, "recognition candidates and beams cannot be combined");
  // character locations of the greedy rec loop (alm_omni_set_rec_locations); they describe this decode or none
  const bool Lc = !points_only && c->rec_locations;
  ALM_REQUIRE(!Lc || Wb == 0, ALM_ERR_INVALID, "character locations and beams cannot be combined");
  if (!points_only) m->rec_lists = {};
  c->timing_valid[1] = false;
  DecodeScope scope(c);
  ALM_CHECK_CUDA(cudaEventRecord(c->ev_t[2], c->stream));

  // ------------------------------------------------------------------ pt loop (transformer.py:102-141)
  const int Tpt = n_prompt + pt_steps;
  const int S = B * P;  // (image, prompt) slots = pt-loop sequences
  int* pt_tok = ws.get<int>(static_cast<size_t>(S) * Tpt);
  float* pt_prob = ws.get<float>(static_cast<size_t>(S) * pt_steps);
  int* finished = ws.get<int>(S);
  int* ntok = ws.get<int>(S);
  {
    std::vector<int> h(static_cast<size_t>(S) * Tpt, 0);
    for (int b = 0; b < B; ++b)
      for (int p = 0; p < P; ++p)
        for (int i = 0; i < n_prompt; ++i)
          h[(static_cast<size_t>(b) * P + p) * Tpt + i] = static_cast<int>(prompts[b * page_stride + p * n_prompt + i]);
    ALM_CHECK_CUDA(cudaMemcpyAsync(pt_tok, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice, c->stream));
    wait_stream(c, c->stream);  // h goes out of scope (this also waits for the encoder)
  }
  fill_i32(c, finished, S, 0);
  fill_i32(c, ntok, S, 0);
  const size_t after_pt_tokens = ws.mark();
  {
    const bool all_done = pt_loop(c, m, hc, 0, B, P, n_prompt, pt_steps, pt_clamped, pt_tok, pt_prob, finished, ntok);
    ALM_REQUIRE(level0 || !pt_clamped || all_done, ALM_ERR_INVALID,
                "an image produced no EOS within the 1024-row position table (the reference raises at transformer.py:312)");
  }
  ALM_CHECK_CUDA(cudaEventRecord(c->ev_t[3], c->stream));
  wait_stream(c, c->stream);
  std::vector<int> h_ntok(S), h_tok(static_cast<size_t>(S) * Tpt), h_fin(level0 ? S : 0);
  std::vector<float> h_prob(static_cast<size_t>(S) * pt_steps);
  ALM_CHECK_CUDA(cudaMemcpyAsync(h_ntok.data(), ntok, S * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  ALM_CHECK_CUDA(cudaMemcpyAsync(h_tok.data(), pt_tok, h_tok.size() * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  ALM_CHECK_CUDA(cudaMemcpyAsync(h_prob.data(), pt_prob, h_prob.size() * sizeof(float), cudaMemcpyDeviceToHost, c->stream));
  if (level0)
    ALM_CHECK_CUDA(cudaMemcpyAsync(h_fin.data(), finished, S * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  if (level0) {  // a saturated sequence ran all pt_steps steps without choosing pt_eos (dense_core.h)
    level0->sat.resize(S);
    for (int q = 0; q < S; ++q) level0->sat[q] = h_fin[q] == 0;
    level0->saturated = std::find(level0->sat.begin(), level0->sat.end(), 1) != level0->sat.end();
    if (level0->saturated) {  // the caller reads the saturated pages in windows: no polygon / recognition loops here
      level0->ntok.swap(h_ntok);
      level0->tok.swap(h_tok);
      ws.release(m->ws_mark);
      return;
    }
  }
  const int maxI = cfg.max_instances;
  // which decoded tokens form (x, y) instances
  std::vector<std::vector<int>> starts(S);
  for (int q = 0; q < S; ++q) {
    int len = h_ntok[q];
    if (len % 2) --len;  // transformer.py:138-139 (applied in both modes by the reference)
    const int* t = &h_tok[static_cast<size_t>(q) * Tpt + n_prompt];
    if (points_only) {  // the raw point sequence is the result (decode_pt_seq alone, transformer.py:102-141)
      n_tok_out[q] = len;
      for (int i = 0; i < len; ++i) {
        pt_tok_out[static_cast<size_t>(q) * cfg.pt_seq_length + i] = t[i];
        if (pt_prob_out) pt_prob_out[static_cast<size_t>(q) * cfg.pt_seq_length + i] = h_prob[static_cast<size_t>(q) * pt_steps + i];
      }
      continue;
    }
    if (!kie) {
      for (int i = 0; i + 1 < len; i += 2) starts[q].push_back(i);
    } else {
      for (int i = 0; i < len;) {  // the walk of decode_vie_pt_poly_rec_seq (transformer.py:148-215)
        if (t[i] < cfg.num_bins && i + 1 <= len - 1 && t[i + 1] < cfg.num_bins) { starts[q].push_back(i); i += 2; }
        else ++i;
      }
      if (n_tok_out) n_tok_out[q] = len;
      for (int i = 0; i < len; ++i) {
        pt_tok_out[static_cast<size_t>(q) * cfg.pt_seq_length + i] = t[i];
        pt_prob_out[static_cast<size_t>(q) * cfg.pt_seq_length + i] = h_prob[static_cast<size_t>(q) * pt_steps + i];
      }
    }
    n_inst[q] = static_cast<int>(starts[q].size());
    ALM_REQUIRE(n_inst[q] <= maxI, ALM_ERR_INVALID, "decoded more points than max_instances");
    for (int n = 0; n < n_inst[q]; ++n) {
      if (inst_pos) inst_pos[static_cast<size_t>(q) * maxI + n] = starts[q][n];
      if (pt) {
        pt[(static_cast<size_t>(q) * maxI + n) * 2] = t[starts[q][n]];
        pt[(static_cast<size_t>(q) * maxI + n) * 2 + 1] = t[starts[q][n] + 1];
      }
    }
  }
  // The poly / rec sequences are [x, y, sos] + generated (transformer.py:252,268): they never see the pt prompt, so
  // every distinct (x, y) of an image is decoded once and its result goes to every slot that holds it.  uniq[b] lists
  // them in first-appearance order over the prompts; slot_inst[q][n] is the entry of instance n of slot q.  With one
  // prompt per image the instances are taken as decoded, so the single-prompt batch shapes stay as they are.
  std::vector<std::vector<std::pair<int, int>>> uniq(B);
  std::vector<std::vector<int>> slot_inst(S);
  if (!points_only) {
    for (int b = 0; b < B; ++b) {
      for (int p = 0; p < P; ++p) {
        const int q = b * P + p;
        const int* t = &h_tok[static_cast<size_t>(q) * Tpt + n_prompt];
        for (int n = 0; n < n_inst[q]; ++n) {
          const std::pair<int, int> xy(t[starts[q][n]], t[starts[q][n] + 1]);
          int e = static_cast<int>(uniq[b].size());
          if (P > 1) e = static_cast<int>(std::find(uniq[b].begin(), uniq[b].end(), xy) - uniq[b].begin());
          if (e == static_cast<int>(uniq[b].size())) uniq[b].push_back(xy);
          slot_inst[q].push_back(e);
        }
      }
    }
  }
  if (points_only) {
    c->timing_valid[1] = true;
    ALM_CHECK_CUDA(cudaEventRecord(c->ev_t[4], c->stream));
    ws.release(m->ws_mark);
    return;
  }
  ws.release(after_pt_tokens);
  poly_rec_loops(c, cfg, hc, P, maxI, uniq, slot_inst, poly, rec, rec_prob);
}

size_t omni_dense_loops(Ctx* c, int32_t* out, size_t elems) {
  OmniModel* m = c->omni;
  ALM_REQUIRE(m != nullptr, ALM_ERR_STATE, "no model loaded");
  const size_t n = m->dense_loops.size();
  if (out == nullptr && elems == 0) return n / 4;  // the count alone
  ALM_REQUIRE(out != nullptr && elems >= n, ALM_ERR_INVALID,
              "loop buffer too small: need " + std::to_string(n) + " elements");
  std::copy(m->dense_loops.begin(), m->dense_loops.end(), out);
  return n / 4;
}

size_t omni_rec_beams(Ctx* c, int64_t* ids, float* probs, float* scores, size_t elems) {
  OmniModel* m = c->omni;
  ALM_REQUIRE(m && !m->rec_lists.beam_ids.empty(), ALM_ERR_STATE,
              "no n-best lists: the last decode ran with alm_omni_set_rec_beams W = 0");
  const size_t n = m->rec_lists.beam_ids.size();
  ALM_REQUIRE(elems >= n, ALM_ERR_INVALID, "n-best buffers too small: need " + std::to_string(n) + " elements");
  std::copy(m->rec_lists.beam_ids.begin(), m->rec_lists.beam_ids.end(), ids);
  std::copy(m->rec_lists.beam_probs.begin(), m->rec_lists.beam_probs.end(), probs);
  std::copy(m->rec_lists.beam_scores.begin(), m->rec_lists.beam_scores.end(), scores);
  return n;
}

size_t omni_rec_locations(Ctx* c, float* out, size_t elems) {
  OmniModel* m = c->omni;
  ALM_REQUIRE(m && !m->rec_lists.rec_loc.empty(), ALM_ERR_STATE,
              "no character locations: the last decode ran with alm_omni_set_rec_locations off");
  const size_t n = m->rec_lists.rec_loc.size();
  ALM_REQUIRE(elems >= n, ALM_ERR_INVALID, "location buffer too small: need " + std::to_string(n) + " elements");
  std::copy(m->rec_lists.rec_loc.begin(), m->rec_lists.rec_loc.end(), out);
  return n;
}

size_t omni_rec_candidates(Ctx* c, int64_t* ids, float* probs, size_t elems) {
  OmniModel* m = c->omni;
  ALM_REQUIRE(m && !m->rec_lists.cand_ids.empty(), ALM_ERR_STATE,
              "no recognition candidates: the last decode ran with alm_omni_set_rec_candidates k = 0");
  const size_t n = m->rec_lists.cand_ids.size();
  ALM_REQUIRE(elems >= n, ALM_ERR_INVALID, "candidate buffers too small: need " + std::to_string(n) + " elements");
  std::copy(m->rec_lists.cand_ids.begin(), m->rec_lists.cand_ids.end(), ids);
  std::copy(m->rec_lists.cand_probs.begin(), m->rec_lists.cand_probs.end(), probs);
  return n;
}

void omni_decode(Ctx* c, const int64_t* pt_prompt, int n_prompt, const alm_decode_cfg& cfg, int32_t* n_inst,
                 int64_t* pt, int64_t* poly, int64_t* rec, float* rec_prob) {
  omni_decode_impl(c, pt_prompt, 0, 1, n_prompt, cfg, false, nullptr, nullptr, nullptr, n_inst, nullptr, pt, poly, rec,
                   rec_prob);
}

void omni_decode_prompts(Ctx* c, const int64_t* prompts, int P, int n_prompt, const alm_decode_cfg& cfg, int32_t* n_inst,
                         int64_t* pt, int64_t* poly, int64_t* rec, float* rec_prob) {
  OmniModel* m = c->omni;
  ALM_REQUIRE(m && m->encoded, ALM_ERR_STATE, "alm_omni_decode_prompts before alm_omni_encode");
  ALM_REQUIRE(P >= 1 && P <= 16, ALM_ERR_INVALID, "prompts per image must be 1..16");
  ALM_REQUIRE(n_prompt >= 1 && n_prompt <= 16, ALM_ERR_INVALID, "pt prompt length");
  for (long i = 0; i < static_cast<long>(m->B) * P * n_prompt; ++i)
    ALM_REQUIRE(prompts[i] >= 0 && prompts[i] < m->V, ALM_ERR_INVALID, "prompt token id out of range");
  omni_decode_impl(c, prompts, static_cast<long>(P) * n_prompt, P, n_prompt, cfg, false, nullptr, nullptr, nullptr, n_inst,
                   nullptr, pt, poly, rec, rec_prob);
}

void omni_decode_kie(Ctx* c, const int64_t* pt_prompt, int n_prompt, const alm_decode_cfg& cfg, int32_t* n_tok,
                     int64_t* pt_tokens, float* pt_probs, int32_t* n_inst, int32_t* inst_pos, int64_t* poly,
                     int64_t* rec, float* rec_prob) {
  omni_decode_impl(c, pt_prompt, 0, 1, n_prompt, cfg, true, n_tok, pt_tokens, pt_probs, n_inst, inst_pos, nullptr, poly,
                   rec, rec_prob);
}

void omni_decode_points(Ctx* c, const int64_t* pt_prompt, int n_prompt, const alm_decode_cfg& cfg, int32_t* n_tok,
                        int64_t* pt_tokens, float* pt_probs) {
  omni_decode_impl(c, pt_prompt, 0, 1, n_prompt, cfg, c->omni && c->omni->vie > 0, n_tok, pt_tokens, pt_probs, nullptr,
                   nullptr, nullptr, nullptr, nullptr, nullptr, true);
}

// The polygon and recognition loops at caller points (alm_omni_decode_at): image b's rows are its count[b] points in
// the caller's order, no dedupe -- the rows omni_decode_impl builds for one prompt per image, so the same points give
// the same Ncap, launches and bits as the decode that produced them.
void omni_decode_at(Ctx* c, const int32_t* xy, const int32_t* count, int cap, const alm_decode_cfg& cfg, int64_t* poly,
                    int64_t* rec, float* rec_prob) {
  OmniModel* m = c->omni;
  ALM_REQUIRE(m && m->encoded, ALM_ERR_STATE, "alm_omni_decode_at before alm_omni_encode");
  ALM_REQUIRE(m->vie == 0, ALM_ERR_INVALID, "alm_omni_decode_at: a KIE checkpoint (its classes come from the point loop)");
  ALM_REQUIRE(cfg.vie_categories == m->vie, ALM_ERR_INVALID, "vie_categories does not match the loaded checkpoint");
  ALM_REQUIRE(m->kv_decoders == 3, ALM_ERR_STATE,
              "the batch was encoded with kv_decoders < 3: only alm_omni_decode_points can run on it");
  ALM_REQUIRE(c->xattn_impl != 1 || m->vt_hi, ALM_ERR_STATE, "xattn_impl 1 must be set before alm_omni_encode");
  ALM_REQUIRE(cap >= 1, ALM_ERR_INVALID, "alm_omni_decode_at: cap must be >= 1");
  ALM_REQUIRE(cfg.poly_length == 32, ALM_ERR_INVALID, "polygon length is fixed at 32 (transformer.py:254)");
  ALM_REQUIRE(cfg.num_bins >= 1 && cfg.num_bins <= m->V, ALM_ERR_INVALID, "num_bins");
  ALM_REQUIRE(cfg.rec_length >= 1 && cfg.rec_length <= 1021, ALM_ERR_INVALID,
              "rec_length must be 1..1021 (the 1024-row position table holds [x, y, sos] + rec_length)");
  const int B = m->B, maxI = std::min(cap, cfg.max_instances);
  for (int b = 0; b < B; ++b) {
    ALM_REQUIRE(count[b] >= 0 && count[b] <= maxI, ALM_ERR_INVALID,
                "alm_omni_decode_at: count[" + std::to_string(b) + "] outside [0, min(cap, max_instances)]");
    for (int n = 0; n < 2 * count[b]; ++n) {
      const int v = xy[static_cast<size_t>(b) * cap * 2 + n];
      ALM_REQUIRE(v >= 0 && v < cfg.num_bins, ALM_ERR_INVALID,
                  "alm_omni_decode_at: page " + std::to_string(b) + " has a bin outside [0, num_bins)");
    }
  }
  check_rec_charset(c, cfg, static_cast<long>(B) * cap);
  std::vector<std::vector<std::pair<int, int>>> uniq(B);
  std::vector<std::vector<int>> slot_inst(B);
  for (int b = 0; b < B; ++b)
    for (int n = 0; n < count[b]; ++n) {
      const int32_t* p = xy + (static_cast<size_t>(b) * cap + n) * 2;
      uniq[b].emplace_back(p[0], p[1]);
      slot_inst[b].push_back(n);
    }
  const size_t rows = static_cast<size_t>(B) * cap;
  std::fill(poly, poly + rows * 32, 0);
  std::fill(rec, rec + rows * cfg.rec_length, 0);
  std::fill(rec_prob, rec_prob + rows * cfg.rec_length, 0.f);
  m->rec_lists = {};
  c->ws.release(m->ws_mark);
  c->timing_valid[1] = false;
  DecodeScope scope(c);
  // no point loop: its phase of alm_omni_last_timing is empty
  ALM_CHECK_CUDA(cudaEventRecord(c->ev_t[2], c->stream));
  ALM_CHECK_CUDA(cudaEventRecord(c->ev_t[3], c->stream));
  const HeadCfg hc{cfg.num_bins, cfg.pt_eos, cfg.rec_eos, cfg.recog_pad, m->vie};
  poly_rec_loops(c, cfg, hc, 1, cap, uniq, slot_inst, poly, rec, rec_prob,
                 c->rec_cs_rows.empty() ? nullptr : c->rec_cs_rows.data(), cap);
}

// Teacher-forced logits for one image: every position of every sequence (Transformer.decode, :74-100).
void omni_decode_logits(Ctx* c, int image, int kind, const int64_t* seq, int n_seq, int len, float* logits) {
  OmniModel* m = c->omni;
  ALM_REQUIRE(m && m->encoded, ALM_ERR_STATE, "alm_omni_decode_logits before alm_omni_encode");
  ALM_REQUIRE(c->xattn_impl != 1 || m->vt_hi, ALM_ERR_STATE, "xattn_impl 1 must be set before alm_omni_encode");
  ALM_REQUIRE(image >= 0 && image < m->B && kind >= 0 && kind < 3 && n_seq > 0 && len > 0 && len <= 1024,
              ALM_ERR_INVALID, "decode_logits arguments");
  ALM_REQUIRE(kind < m->kv_decoders, ALM_ERR_STATE, "the batch was encoded without this decoder's K/V cache (kv_decoders)");
  Arena& ws = c->ws;
  ws.release(m->ws_mark);
  std::vector<int> h(static_cast<size_t>(n_seq) * len);
  for (size_t i = 0; i < h.size(); ++i) {
    ALM_REQUIRE(seq[i] >= 0 && seq[i] < m->V, ALM_ERR_INVALID, "token id out of range");
    h[i] = static_cast<int>(seq[i]);
  }
  int* tok = ws.get<int>(h.size());
  ALM_CHECK_CUDA(cudaMemcpyAsync(tok, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice, c->stream));
  StepBufs u = alloc_decode(c, m, 1, 1, n_seq, len, false, image);
  fill_i32(c, u.all.tpos, 1, 0);
  for (int t = 0; t < len; ++t) {
    decoder_step(c, m, kind, u, &tok, &len, image, 1, true);
    add_i32(c, u.all.tpos, 1);
    // logits [n_seq, len, V] <- step t rows
    ALM_CHECK_CUDA(cudaMemcpy2DAsync(logits + static_cast<size_t>(t) * m->V, static_cast<size_t>(len) * m->V * sizeof(float),
                                     u.all.logits, static_cast<size_t>(m->V) * sizeof(float), static_cast<size_t>(m->V) * sizeof(float),
                                     n_seq, cudaMemcpyDeviceToHost, c->stream));
  }
  ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  ws.release(m->ws_mark);
}

// ================================================================================================ dense pages
// Pages with more words than one point sequence holds, read in the training grids' spatial windows (DESIGN 4.16;
// rule: dense_core.h).
namespace {

// maximal runs [first, first + count) of consecutive pages with want[b]
std::vector<std::pair<int, int>> page_runs(const std::vector<uint8_t>& want) {
  std::vector<std::pair<int, int>> runs;
  for (int b = 0; b < static_cast<int>(want.size());) {
    if (!want[b]) { ++b; continue; }
    int e = b;
    while (e < static_cast<int>(want.size()) && want[e]) ++e;
    runs.emplace_back(b, e - b);
    b = e;
  }
  return runs;
}

// Pages img0 .. img0 + nimg - 1 read at grid (nx, ny): the P = nx ny window prompts of every page through one point
// loop, then dense_own_kernel.  pts[b * kMaxWindows + w] gets window w's owned points, sat the same slot's flag.
// The decode kernels take a contiguous slice of the encoded batch, so the caller passes runs of consecutive pages:
// pages outside the slice add no query rows and their K_c / V_c are not streamed.
void read_windows(Ctx* c, OmniModel* m, const HeadCfg& hc, const int64_t* prompt, int n_prompt, int pt_steps, int nx,
                  int ny, int img0, int nimg, std::vector<Points>* pts, uint8_t* sat) {
  Arena& ws = c->ws;
  const size_t mark = ws.mark();
  const int P = nx * ny, S = nimg * P, Tpt = n_prompt + pt_steps, nb = hc.num_bins;
  const int max_pts = std::max(1, pt_steps / 2);
  std::vector<int> h(static_cast<size_t>(S) * Tpt, 0);
  for (int q = 0; q < S; ++q) {
    int* row = &h[static_cast<size_t>(q) * Tpt];
    for (int i = 0; i < n_prompt; ++i) row[i] = static_cast<int>(prompt[i]);
    dense_core::window(nb, nx, ny, q % P, row);  // the box tokens 0..3; character range and pt_sos kept
  }
  int* pt_tok = ws.get<int>(h.size());
  float* pt_prob = ws.get<float>(static_cast<size_t>(S) * pt_steps);
  int* finished = ws.get<int>(S);
  int* ntok = ws.get<int>(S);
  int* xy = ws.get<int>(static_cast<size_t>(S) * max_pts * 2);
  int* own = ws.get<int>(2 * static_cast<size_t>(S));
  ALM_CHECK_CUDA(cudaMemcpyAsync(pt_tok, h.data(), h.size() * sizeof(int), cudaMemcpyHostToDevice, c->stream));
  fill_i32(c, finished, S, 0);
  fill_i32(c, ntok, S, 0);
  m->dense_loops.insert(m->dense_loops.end(), {0, img0, nimg, P});
  pt_loop(c, m, hc, img0, nimg, P, n_prompt, pt_steps, false, pt_tok, pt_prob, finished, ntok);
  dense_own(c, S, P, pt_tok, Tpt, n_prompt, ntok, finished, nb, nx, ny, max_pts, xy, own);
  std::vector<int> h_own(2 * static_cast<size_t>(S)), h_xy(static_cast<size_t>(S) * max_pts * 2);
  ALM_CHECK_CUDA(cudaMemcpyAsync(h_own.data(), own, h_own.size() * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  ALM_CHECK_CUDA(cudaMemcpyAsync(h_xy.data(), xy, h_xy.size() * sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  ALM_CHECK_CUDA(cudaStreamSynchronize(c->stream));
  for (int q = 0; q < S; ++q) {
    const int b = img0 + q / P, w = q % P;
    Points& p = (*pts)[static_cast<size_t>(b) * dense_core::kMaxWindows + w];
    p.clear();
    for (int k = 0; k < h_own[2 * q]; ++k)
      p.emplace_back(h_xy[(static_cast<size_t>(q) * max_pts + k) * 2], h_xy[(static_cast<size_t>(q) * max_pts + k) * 2 + 1]);
    sat[static_cast<size_t>(b) * dense_core::kMaxWindows + w] = static_cast<uint8_t>(h_own[2 * q + 1]);
  }
  ws.release(mark);
}

// Polygon and recognition loops (transformer.py:249-284) of the distinct points uniq[b] of every page, in passes of at
// most `budget` rows: a pass is a run of consecutive pages that still have points, Ncap rows per page (the run's
// largest remainder, at most budget / pages), so a page whose points are done adds no rows and streams no K_c / V_c.
// Per point: poly [32], rec / prob [rec_length], in uniq order.
void poly_rec_passes(Ctx* c, OmniModel* m, const alm_decode_cfg& cfg, const HeadCfg& hc, const std::vector<Points>& uniq,
                     long budget, std::vector<std::vector<int>>* poly, std::vector<std::vector<int>>* rec,
                     std::vector<std::vector<float>>* prob) {
  const int B = m->B, L1 = cfg.poly_length, L2 = cfg.rec_length;
  Arena& ws = c->ws;
  for (int b = 0; b < B; ++b) {
    (*poly)[b].assign(uniq[b].size() * L1, 0);
    (*rec)[b].assign(uniq[b].size() * L2, 0);
    (*prob)[b].assign(uniq[b].size() * L2, 0.f);
  }
  std::vector<int> next(B, 0);
  for (;;) {
    std::vector<uint8_t> left(B);
    for (int b = 0; b < B; ++b) left[b] = next[b] < static_cast<int>(uniq[b].size());
    const std::vector<std::pair<int, int>> runs = page_runs(left);
    if (runs.empty()) break;
    for (const auto& run : runs) {
      const int i0 = run.first, n = run.second;
      long most = 0;
      for (int b = i0; b < i0 + n; ++b) most = std::max<long>(most, static_cast<long>(uniq[b].size()) - next[b]);
      const int Ncap = static_cast<int>(std::min<long>(most, std::max<long>(1, budget / n)));
      m->dense_loops.insert(m->dense_loops.end(), {1, i0, n, Ncap});
      std::vector<Points> pts(n);  // the pass's rows of each page: its next Ncap points
      for (int b = i0; b < i0 + n; ++b)
        pts[b - i0].assign(uniq[b].begin() + next[b], uniq[b].begin() + std::min<size_t>(uniq[b].size(), next[b] + Ncap));
      const size_t mark = ws.mark();
      const PolyRec r = poly_rec(c, cfg, hc, i0, pts, Ncap, nullptr);
      for (int b = i0; b < i0 + n; ++b) {
        for (size_t j = 0; j < pts[b - i0].size(); ++j) {
          const size_t row = static_cast<size_t>(b - i0) * Ncap + j, e = next[b] + j;
          std::copy_n(r.tok[1].begin() + row * (3 + L1) + 3, L1, (*poly)[b].begin() + e * L1);
          std::copy_n(r.tok[2].begin() + row * (3 + L2) + 3, L2, (*rec)[b].begin() + e * L2);
          std::copy_n(r.prob[2].begin() + row * L2, L2, (*prob)[b].begin() + e * L2);
        }
        next[b] += static_cast<int>(pts[b - i0].size());
      }
      ws.release(mark);
    }
  }
}

}  // namespace

void omni_decode_dense(Ctx* c, const int64_t* prompt, int n_prompt, const alm_decode_cfg& cfg, int nx, int ny,
                       double iou, int cap, int32_t* n_inst, int64_t* pt, int64_t* poly, int64_t* rec, float* rec_prob,
                       int32_t* window, int32_t* grid, uint8_t* saturated) {
  using dense_core::kMaxWindows;
  OmniModel* m = c->omni;
  const std::string fn = "alm_omni_decode_dense: ";
  ALM_REQUIRE(m && m->encoded, ALM_ERR_STATE, fn + "no encoded batch");
  ALM_REQUIRE(m->vie == 0, ALM_ERR_INVALID, fn + "a KIE checkpoint has no spatial windows (text spotting only)");
  ALM_REQUIRE((nx == 0 && ny == 0) || dense_core::trained_grid(nx, ny), ALM_ERR_INVALID,
              fn + "grid must be (0, 0) for 'auto' or (nx, ny) with nx, ny in 1..3, the trained grids");
  ALM_REQUIRE(n_prompt >= 5 && n_prompt <= 16, ALM_ERR_INVALID, fn + "the prompt must hold a box: 5..16 tokens");
  for (int i = 0; i < n_prompt; ++i)
    ALM_REQUIRE(prompt[i] >= 0 && prompt[i] < m->V, ALM_ERR_INVALID, fn + "prompt token id out of range");
  const int nb = cfg.num_bins;
  ALM_REQUIRE(nb >= 3 && prompt[0] == 0 && prompt[1] == 0 && prompt[2] == nb - 1 && prompt[3] == nb - 1,
              ALM_ERR_INVALID, fn + "the prompt's box must be the whole page (0, 0, num_bins - 1, num_bins - 1)");
  ALM_REQUIRE(std::isfinite(iou) && iou > 0.0 && iou <= 1.0, ALM_ERR_INVALID, fn + "iou must be in (0, 1]");
  ALM_REQUIRE(c->rec_topk == 0 && c->rec_beams == 0 && !c->rec_locations, ALM_ERR_INVALID,
              fn + "recognition candidates, beams and character locations cannot be combined with dense decoding");
  ALM_REQUIRE(cfg.pt_seq_length >= 1, ALM_ERR_INVALID, fn + "pt_seq_length");
  ALM_REQUIRE(cfg.vie_categories == m->vie, ALM_ERR_INVALID, fn + "vie_categories does not match the loaded checkpoint");
  ALM_REQUIRE(m->kv_decoders == 3, ALM_ERR_STATE, fn + "the batch was encoded with kv_decoders < 3");
  ALM_REQUIRE(cfg.poly_length == 32, ALM_ERR_UNSUPPORTED, fn + "polygon length is fixed at 32 (transformer.py:254)");
  ALM_REQUIRE(c->xattn_impl != 1 || m->vt_hi, ALM_ERR_STATE, fn + "xattn_impl 1 must be set before alm_omni_encode");
  const int pt_steps = std::min(cfg.pt_seq_length, 1025 - n_prompt), per_seq = pt_steps / 2;
  ALM_REQUIRE(cfg.max_instances >= per_seq, ALM_ERR_INVALID, fn + "max_instances < pt_seq_length / 2");
  const long most = static_cast<long>(nx ? nx * ny : kMaxWindows) * per_seq;
  ALM_REQUIRE(cap >= 1 && cap >= most, ALM_ERR_INVALID,
              fn + "cap is below what the grid can produce: " + std::to_string(most) + " rows per page");
  check_rec_charset(c, cfg, -1);  // honoured by every polygon / recognition pass, set 0 on every row

  // the preamble of every decode entry: a fresh workspace after the encoded state, and no candidate / n-best / location
  // lists (they describe the last decode or none; dense decoding makes none)
  c->ws.release(m->ws_mark);
  m->rec_lists = {};
  m->dense_loops.clear();
  const int B = m->B, L = cfg.rec_length;
  const size_t W = kMaxWindows;
  std::optional<DecodeScope> scope;  // the decode-loop settings (as omni_decode_impl) for the loops below
  std::fill(saturated, saturated + B * W, uint8_t(0));
  std::vector<Points> pts(B * W);      // [page][window]: owned points in decode order
  std::vector<int> gx(B, 1), gy(B, 1);  // each page's grid
  HeadCfg hc{cfg.num_bins, cfg.pt_eos, cfg.rec_eos, cfg.recog_pad, m->vie};
  if (nx == 0) {
    // level 0: decode itself; when nothing saturates its outputs are the result, in decode's launches and bits
    alm_decode_cfg lay = cfg;
    lay.max_instances = cap;
    Level0 l0;
    omni_decode_impl(c, prompt, 0, 1, n_prompt, lay, false, nullptr, nullptr, nullptr, n_inst, nullptr, pt, poly, rec,
                     rec_prob, false, &l0);
    for (int b = 0; b < B; ++b) {
      grid[2 * b] = grid[2 * b + 1] = 1;
      saturated[b * W] = l0.sat[b];
    }
    if (!l0.saturated) {
      for (int b = 0; b < B; ++b) std::fill(window + static_cast<size_t>(b) * cap, window + (b + 1L) * cap, 0);
      return;
    }
    const int Tpt = n_prompt + pt_steps;
    std::vector<uint8_t> again(B);
    for (int b = 0; b < B; ++b) {
      again[b] = l0.sat[b];
      if (again[b]) continue;
      const int* t = &l0.tok[static_cast<size_t>(b) * Tpt + n_prompt];
      for (int i = 0; i + 1 < (l0.ntok[b] & ~1); i += 2) pts[b * W].emplace_back(t[i], t[i + 1]);
    }
    scope.emplace(c);
    for (int level = 2; level <= 3; ++level) {  // 2 x 2 for the saturated pages, 3 x 3 for those still saturated
      for (const auto& run : page_runs(again))
        read_windows(c, m, hc, prompt, n_prompt, pt_steps, level, level, run.first, run.second, &pts, saturated);
      for (int b = 0; b < B; ++b) {
        if (!again[b]) continue;
        gx[b] = gy[b] = level;
        again[b] = std::find(saturated + b * W, saturated + b * W + level * level, 1) != saturated + b * W + level * level;
        if (level == 2 && again[b]) std::fill(saturated + b * W, saturated + (b + 1) * W, uint8_t(0));
      }
    }
  } else {
    scope.emplace(c);
    read_windows(c, m, hc, prompt, n_prompt, pt_steps, nx, ny, 0, B, &pts, saturated);
    std::fill(gx.begin(), gx.end(), nx);
    std::fill(gy.begin(), gy.end(), ny);
  }
  for (int b = 0; b < B; ++b) {
    grid[2 * b] = gx[b];
    grid[2 * b + 1] = gy[b];
  }

  // every distinct point of a page decoded once (the windows partition the page; a point repeated within a window
  // shares its entry), in passes of at most the rows of the largest decode of the batch, B x max_instances
  std::vector<Points> uniq(B);
  std::vector<std::vector<int>> entry(B * W);
  for (int b = 0; b < B; ++b) {
    std::unordered_map<int64_t, int> seen;  // (x, y) -> its entry: linear in the page's points
    for (int w = 0; w < gx[b] * gy[b]; ++w)
      for (const auto& xy : pts[b * W + w]) {
        const int64_t key = (static_cast<int64_t>(xy.first) << 32) | static_cast<uint32_t>(xy.second);
        const auto it = seen.emplace(key, static_cast<int>(uniq[b].size())).first;
        if (it->second == static_cast<int>(uniq[b].size())) uniq[b].push_back(xy);
        entry[b * W + w].push_back(it->second);
      }
  }
  std::vector<std::vector<int>> h_poly(B), h_rec(B);
  std::vector<std::vector<float>> h_prob(B);
  poly_rec_passes(c, m, cfg, hc, uniq, static_cast<long>(B) * cfg.max_instances, &h_poly, &h_rec, &h_prob);

  // rows per (page, window) in decode order; pages read in windows merged on the device (turn_core.h's rule over
  // nr readings), a page with one reading taken as it is
  int nr = 1;
  std::vector<int> merged;  // pages with more than one window
  for (int b = 0; b < B; ++b)
    if (gx[b] * gy[b] > 1) {
      merged.push_back(b);
      nr = std::max(nr, gx[b] * gy[b]);
    }
  auto put = [&](int b, int r, int w, double x, double y, const double* pv, const int64_t* rc, const float* pr) {
    const size_t o = static_cast<size_t>(b) * cap + r;
    pt[o * 2] = static_cast<int64_t>(x);
    pt[o * 2 + 1] = static_cast<int64_t>(y);
    for (int k = 0; k < 32; ++k) poly[o * 32 + k] = static_cast<int64_t>(pv[k]);
    for (int k = 0; k < L; ++k) { rec[o * L + k] = rc[k]; rec_prob[o * L + k] = pr[k]; }
    window[o] = w;
  };
  auto row_of = [&](int b, int w, int i, double* xy, double* pv, int64_t* rc, float* pr) {
    const int e = entry[b * W + w][i];
    xy[0] = uniq[b][e].first;
    xy[1] = uniq[b][e].second;
    for (int k = 0; k < 32; ++k) pv[k] = h_poly[b][static_cast<size_t>(e) * 32 + k];
    for (int k = 0; k < L; ++k) { rc[k] = h_rec[b][static_cast<size_t>(e) * L + k]; pr[k] = h_prob[b][static_cast<size_t>(e) * L + k]; }
  };
  for (int b = 0; b < B; ++b) {
    std::fill(window + static_cast<size_t>(b) * cap, window + (b + 1L) * cap, 0);
    if (gx[b] * gy[b] > 1) continue;
    n_inst[b] = static_cast<int>(entry[b * W].size());
    for (int i = 0; i < n_inst[b]; ++i) {
      double xy[2], pv[32];
      std::vector<int64_t> rc(L);
      std::vector<float> pr(L);
      row_of(b, 0, i, xy, pv, rc.data(), pr.data());
      put(b, i, 0, xy[0], xy[1], pv, rc.data(), pr.data());
    }
  }
  if (merged.empty()) return;
  const int np = static_cast<int>(merged.size());
  std::vector<int> count(static_cast<size_t>(np) * nr, 0), offset(count.size(), 0);
  long N = 0;
  for (int j = 0; j < np; ++j)
    for (int w = 0; w < nr; ++w) {
      const int b = merged[j];
      offset[j * nr + w] = static_cast<int>(N);
      count[j * nr + w] = w < gx[b] * gy[b] ? static_cast<int>(entry[b * W + w].size()) : 0;
      N += count[j * nr + w];
    }
  const size_t rows = static_cast<size_t>(std::max<long>(N, 1));
  std::vector<double> d_pts(rows * 2), d_polys(rows * 32), o_pts(rows * 2), o_polys(rows * 32);
  std::vector<int64_t> d_rec(rows * L), o_rec(rows * L);
  std::vector<float> d_prob(rows * L), o_prob(rows * L);
  std::vector<int> src(rows * 2), pc(np), po(np);
  for (int j = 0; j < np; ++j)
    for (int w = 0; w < nr; ++w)
      for (int i = 0; i < count[j * nr + w]; ++i) {
        const size_t n = static_cast<size_t>(offset[j * nr + w]) + i;
        row_of(merged[j], w, i, &d_pts[n * 2], &d_polys[n * 32], &d_rec[n * L], &d_prob[n * L]);
      }
  reading_merge(c, np, nr, count.data(), offset.data(), L, cfg.recog_pad, cfg.rec_eos, iou, d_pts.data(),
                d_polys.data(), d_rec.data(), d_prob.data(),
                MergeRows{pc.data(), po.data(), o_pts.data(), o_polys.data(), o_rec.data(), o_prob.data(), src.data()});
  for (int j = 0; j < np; ++j) {
    const int b = merged[j];
    n_inst[b] = pc[j];
    for (int r = 0; r < pc[j]; ++r) {
      const size_t n = static_cast<size_t>(po[j]) + r;
      put(b, r, src[n * 2], o_pts[n * 2], o_pts[n * 2 + 1], &o_polys[n * 32], &o_rec[n * L], &o_prob[n * L]);
    }
  }
}

}  // namespace alm
