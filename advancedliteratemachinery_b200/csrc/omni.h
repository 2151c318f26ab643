// OmniParser model state (weights + per-batch encode/decode buffers) and kernel wrappers.
#pragma once
#include "alm_internal.h"

namespace alm {

struct HeadCfg {
  int num_bins, pt_eos, rec_eos, recog_pad, vie;
  // caller character sets of the rec loop (alm_omni_set_rec_charset), null when none is in force: cs_allowed uint8
  // [n_sets][recog_pad - num_bins - 1] (1 = chars[i] allowed), cs_set int32 [instance] the set of each instance (null:
  // set 0 for every instance); the beam rows of an instance share its set
  const uint8_t* cs_allowed = nullptr;
  const int* cs_set = nullptr;
};

struct LNW {
  float* g = nullptr;
  float* b = nullptr;
};
struct Lin {
  SplitW w;
  float* b = nullptr;
  float* wf = nullptr;  // exact fp32 [N,K] copy (decoder weights only): the skinny M <= 32 decode path
};

struct SwinBlockW {
  LNW n1, n2;
  Lin qkv, proj, fc1, fc2;
  float* bias_dense = nullptr;  // [heads,49,49] = table[index]  (swin_transformer.py:133-135)
};
struct SwinStageW {
  std::vector<SwinBlockW> blocks;
  LNW out_norm;   // norm{s}
  LNW merge_norm;  // downsample.norm
  SplitW merge_red;
};
struct DecLayerW {
  LNW n1, n2, n3;
  Lin sa_qk;   // rows [0,1024) of self_attn.in_proj (q then k)
  Lin sa_v;    // rows [1024,1536)
  float* sa_qkv_f = nullptr;  // exact fp32 packed in_proj [1536,512] + bias [1536] (skinny decode path)
  float* sa_qkv_b = nullptr;
  Lin sa_out;
  Lin ca_q;    // rows [0,512) of multihead_attn.in_proj
  Lin ca_out;
  Lin l1, l2;
};

struct OmniModel {
  int V = 0;
  int vie = 0;
  Lin patch;
  LNW patch_norm;
  SwinStageW stage[4];
  SplitW fpn[4];  // fpn_in[0..3] : c5,c4,c3,c2
  Lin inproj;
  float* dim_t = nullptr;  // [256]
  // decoder
  float* word_emb = nullptr;
  float* pos_emb[3] = {nullptr, nullptr, nullptr};  // pt, poly, rec
  LNW emb_norm;
  DecLayerW dec[3][4];
  LNW dec_norm[3];
  Lin ca_k_all;  // [12*512, 512]  rows (d*4+l)*512..: cross-attn K projections of all decoder layers
  Lin ca_v_all;  // [12*512, 512]
  Lin head[3][3];

  // ---- state of the last alm_omni_encode -------------------------------------------------------
  bool encoded = false;
  int kv_decoders = 3;  // decoders whose K/V caches the last encode filled
  int B = 0, H = 0, W = 0;
  int Hs[4] = {0, 0, 0, 0}, Ws[4] = {0, 0, 0, 0};
  int mh = 0, mw = 0, M = 0, Mpad = 0;  // pages of different sizes: mh = mw = 0, M = largest page's key count
  std::vector<int> page_mh, page_mw;     // memory grid of every page (both encodes)
  bool mixed = false;                    // pages of different sizes (alm_omni_encode_pages): memory rows at stride M
  std::vector<int> page_keys;            // mixed: live keys mh_b * mw_b per page (host copy of key_len)
  int* key_len = nullptr;                // mixed: device [B] live keys per page
  int* kb_off = nullptr;                 // mixed: device [B + 1] running sum of ceil(key_len / 64)
  float* feat[4] = {nullptr, nullptr, nullptr, nullptr};  // LN'd stage outputs, NHWC fp32
  float* memory = nullptr;                                // [B*M,512]
  float* pos = nullptr;                                   // [B*M,512]
  uint8_t* kpm = nullptr;                                 // [B*M]
  bf16 *kc_hi = nullptr, *kc_lo = nullptr;                // [B, 12 (dec,layer), 8 heads, M, 64]
  bf16 *vc_hi = nullptr, *vc_lo = nullptr;                // [B, 12 (dec,layer), 8 heads, M, 64]
  bf16 *vt_hi = nullptr, *vt_lo = nullptr;                // [B, 6144, Mpad] (only for the unfused debug path, xattn_impl 1)
  size_t ws_mark = 0;                                     // arena offset after the encode-persistent buffers
  // side lists of the last decode that ran the rec loop, each empty unless its option was on
  struct RecLists {
    // candidates (Ctx::rec_topk > 0): [slot][max_inst][rec_length][k]
    std::vector<int64_t> cand_ids;
    std::vector<float> cand_probs;
    // n-best lists (Ctx::rec_beams > 0): ids / probs [slot][max_inst][W][rec_length], scores [slot][max_inst][W]
    std::vector<int64_t> beam_ids;
    std::vector<float> beam_probs, beam_scores;
    // character locations (Ctx::rec_locations): [slot][max_inst][rec_length][5] = cx, cy, sxx, sxy, syy in
    // encoder-input pixels
    std::vector<float> rec_loc;
  } rec_lists;
  // the loops of the last alm_omni_decode_dense beyond level 0, [n][4] = (kind, img0, nimg, per page): kind 0 a window
  // point loop with `per page` = P window prompts, kind 1 a polygon / recognition pass of `per page` = Ncap rows
  std::vector<int> dense_loops;
  int* d_page_mw = nullptr;  // device copy of page_mw (encode-persistent)
  // captured decode-step graphs, keyed by everything that determines the launch sequence and its pointers
  struct StepGraph { cudaGraphExec_t exec; long launches; };
  std::map<std::vector<long>, StepGraph> step_graphs;
  ~OmniModel() {
    for (auto& kv : step_graphs) cudaGraphExecDestroy(kv.second.exec);
  }
};

void omni_load(Ctx* c, int kind, const std::map<std::string, HostTensor>& t);
// token grids Hs[s] x Ws[s] of the four Swin stages of an H x W page (patch embed, then three ceil-halving merges)
void stage_grid(int H, int W, int* Hs, int* Ws);
// dim_t[256] of the sine position embedding (position_embedding.py:35-36): 10000^(2 floor(i / 2) / 256)
std::vector<float> sine_dim_t();
// a second execution context over the same device weights: weight pointers copied, per-batch state fresh
OmniModel* omni_share(const OmniModel* owner);
void omni_encode(Ctx* c, const float* img_dev, const uint8_t* mask_dev, int B, int H, int W);
// pages of different sizes: page b is the top-left heights[b] x widths[b] of slot b of img [B,3,Hc,Wc], encoded alone
void omni_encode_pages(Ctx* c, const float* img_dev, int B, int Hc, int Wc, const int* heights, const int* widths);
void omni_decode(Ctx* c, const int64_t* pt_prompt, int n_prompt, const alm_decode_cfg& cfg, int32_t* n_inst,
                 int64_t* pt, int64_t* poly, int64_t* rec, float* rec_prob);
// prompts int64 [B][P][n_prompt]; outputs per (image, prompt) slot, in the layout of omni_decode with B * P images
void omni_decode_prompts(Ctx* c, const int64_t* prompts, int P, int n_prompt, const alm_decode_cfg& cfg, int32_t* n_inst,
                         int64_t* pt, int64_t* poly, int64_t* rec, float* rec_prob);
void omni_decode_kie(Ctx* c, const int64_t* pt_prompt, int n_prompt, const alm_decode_cfg& cfg, int32_t* n_tok,
                     int64_t* pt_tokens, float* pt_probs, int32_t* n_inst, int32_t* inst_pos, int64_t* poly,
                     int64_t* rec, float* rec_prob);
// polygon and recognition loops at caller points: xy int32 [B][cap][2] bins, count int32 [B]; outputs [B][cap][..]
void omni_decode_at(Ctx* c, const int32_t* xy, const int32_t* count, int cap, const alm_decode_cfg& cfg, int64_t* poly,
                    int64_t* rec, float* rec_prob);
void omni_decode_points(Ctx* c, const int64_t* pt_prompt, int n_prompt, const alm_decode_cfg& cfg, int32_t* n_tok,
                        int64_t* pt_tokens, float* pt_probs);
// Dense pages read in spatial windows (DESIGN 4.16; rule: dense_core.h).  (nx, ny) = (0, 0): grid 'auto'.  Outputs per
// page b at cap rows: n_inst [B], pt [B][cap][2], poly [B][cap][32], rec / rec_prob [B][cap][rec_length], window
// [B][cap], grid [B][2], saturated [B][9].
void omni_decode_dense(Ctx* c, const int64_t* prompt, int n_prompt, const alm_decode_cfg& cfg, int nx, int ny,
                       double iou, int cap, int32_t* n_inst, int64_t* pt, int64_t* poly, int64_t* rec, float* rec_prob,
                       int32_t* window, int32_t* grid, uint8_t* saturated);
// loops of the last omni_decode_dense into out [n][4] (elems = its capacity; out NULL and elems 0: the count alone);
// returns n
size_t omni_dense_loops(Ctx* c, int32_t* out, size_t elems);
void omni_decode_logits(Ctx* c, int image, int kind, const int64_t* seq, int n_seq, int len, float* logits);
// candidates of the last decode (Ctx::rec_topk > 0) into ids / probs [slot][max_inst][rec_length][k]; returns the count
size_t omni_rec_candidates(Ctx* c, int64_t* ids, float* probs, size_t elems);
// n-best lists of the last decode (Ctx::rec_beams > 0): ids / probs [slot][max_inst][W][rec_length] (elems = their
// capacity), scores [slot][max_inst][W]; returns the id count
size_t omni_rec_beams(Ctx* c, int64_t* ids, float* probs, float* scores, size_t elems);
// character locations of the last decode (Ctx::rec_locations) into out [slot][max_inst][rec_length][5]; returns the count
size_t omni_rec_locations(Ctx* c, float* out, size_t elems);

// kernels (omni_kernels.cu)
void window_map(Ctx* c, int* map, int B, int H, int W, int nWh, int nWw, int shift);
void merge_map(Ctx* c, int* map, int B, int H, int W, int H2, int W2);
void nearest_map(Ctx* c, int* map, int B, int Hd, int Wd, int Hs, int Ws);
void fpn_assemble(Ctx* c, const float* p2, const float* p3, const float* p4, const float* p5, int B, const int* Hs,
                  const int* Ws, int Ho, int Wo, bf16* hi, bf16* lo);
void sine_pos(Ctx* c, const uint8_t* mask, int B, int H, int W, int h, int w, const float* dim_t, float* pos,
              uint8_t* kpm, float* scratch);
void embed_ln(Ctx* c, const int* tokens, int tstride, const int* tptr, int S, const float* word_emb,
              const float* pos_emb, const float* gamma, const float* beta, float* x, float* qpos, int S_half = 0,
              const int* tokens2 = nullptr, int tstride2 = 0, const float* pos_emb2 = nullptr, float* qpos2 = nullptr);
// anc (beam search, NULL otherwise): int32 [S][Tmax], position j < t of sequence s is cached in row anc[s][j]
void self_attn_step(Ctx* c, const float* qk, const float* vnew, float* kc, float* vc, int S, const int* tptr, int Tmax,
                    bf16* out_hi, bf16* out_lo, float* out_f32 = nullptr, int ld_qk = 1024, int ld_v = 512,
                    const int* anc = nullptr);
void head_select(Ctx* c, const float* logits, int S, int V, int nsoft, int phase, const HeadCfg& cfg, int* tokens,
                 int tstride, const int* tptr, int n_prompt_m1, float* probs, int pstride, int* finished, int* ntok,
                 int seqs_per_image);
// the recognition step (phase 2) of head_select that also writes the k <= 8 most likely allowed classes and their
// probabilities at cand_ids / cand_probs [s * cand_stride + gen_index * k + i]
void head_select_topk(Ctx* c, const float* logits, int S, int V, int nsoft, const HeadCfg& cfg, int* tokens, int tstride,
                      const int* tptr, int n_prompt_m1, float* probs, int pstride, int k, int* cand_ids,
                      float* cand_probs, int cand_stride);
// One beam-search recognition step over G groups of W adjacent rows (omni_kernels.cu: beam_select_kernel).  score [G*W]
// f32 and blen [G*W] int32 carry the hypotheses' state between steps, anc int32 [G*W][Tmax] their ancestry.
void beam_select(Ctx* c, const float* logits, int G, int W, int V, int nsoft, const HeadCfg& cfg, int* tokens, int tstride,
                 const int* tptr, int n_prompt_m1, float* probs, int pstride, float* score, int* blen, int* anc, int Tmax);
void anc_identity(Ctx* c, int* anc, int S, int Tmax);
// n-best lists of the beam loop, ranked by score / len^alpha: ids / probs [G][W][L] (generated positions t0..t0+L-1),
// scores [G][W]
void beam_backtrace(Ctx* c, const int* tokens, int tstride, const float* probs, int pstride, const float* score,
                    const int* blen, const int* anc, int Tmax, int G, int W, int L, int t0, float alpha, int* out_ids,
                    float* out_probs, float* out_scores);
void cross_attn_q1(Ctx* c, const float* q, const bf16* kc_hi, const bf16* kc_lo, const bf16* vt_hi, const bf16* vt_lo,
                   const uint8_t* kpm, int nimg, int M, int Mpad, float* partial, int* counters, int nsplit,
                   bf16* out_hi, bf16* out_lo, float* out_f32 = nullptr);
int cross_attn_q1_splits(Ctx* c, int nimg, int M);
// fused multi-query cross-attention (xattn.cu): Ncap query rows per image against the cached K_c / V_c^T.
// Images are M keys apart in the caches.  Per-image live-key counts (optional; pages of different sizes): key_len
// host [nimg] for the plan, and on the device key_len [nimg] with kb_off [nimg + 1] = running sum of
// ceil(key_len / 64); keys >= key_len[img] are neither streamed beyond their 64-key block nor allowed into the output.
long cross_attn_key_blocks(int nimg, int M, const int* key_len, int* max_blocks);
void cross_attn_mq_plan(Ctx* c, int nimg, int Ncap, int M, int* grid, int* max_parts, int* pairs,
                        const int* key_len = nullptr);
size_t cross_attn_mq_partial_floats(int pairs, int max_parts);
void cross_attn_mq(Ctx* c, const bf16* q_hi, const bf16* q_lo, const float* q_f32, int nimg, int Ncap, const bf16* kc_hi,
                   const bf16* kc_lo, const bf16* vc_hi, const bf16* vc_lo, const uint8_t* kpm, int M,
                   const int* key_len, const int* kb_off, int grid, int max_parts, float* partial, int* counters,
                   bf16* out_hi, bf16* out_lo, float* out_f32);
// experimental TMA + mbarrier variant (xattn_tma.cu, "xattn_impl" 2)
void cross_attn_tma_plan(Ctx* c, int nimg, int Ncap, int M, int* grid, int* max_parts, int* pairs,
                         const int* key_len = nullptr);
void cross_attn_tma(Ctx* c, const bf16* q_hi, const bf16* q_lo, const float* q_f32, int nimg, int Ncap, const bf16* kc_hi,
                    const bf16* kc_lo, const bf16* vc_hi, const bf16* vc_lo, long slices, int z0, const uint8_t* kpm, int M,
                    const int* key_len, const int* kb_off, int grid, int max_parts, float* partial, int* counters,
                    bf16* out_hi, bf16* out_lo, float* out_f32);
// Character locations (xattn_loc.cu): per query row the centroid and central second moments (cx, cy, sxx, sxy, syy)
// of the head-averaged softmax((q_h / 8) K_h^T) over the key positions (16 c + 8, 16 r + 8), r, c = k / mw, k % mw
// of the image's grid width page_mw[img] (device [nimg]).  kc_hi / kc_lo point at the layer's slice as in
// cross_attn_mq; key_len (device, optional) and kpm mask keys like the cross-attention.  Row s of step
// gen = *tpos - t0 (gen 0 without tpos) goes to out[(s * L + gen) * 5].  The plan gives the key splits per head,
// the partial buffer size and the counter count (counters zeroed once; every launch leaves them zero).
void rec_locate_plan(Ctx* c, int nimg, int Ncap, int M, const int* key_len, int* ks, size_t* partial_floats, int* groups);
void rec_locate(Ctx* c, const bf16* q_hi, const bf16* q_lo, const float* q_f32, int nimg, int Ncap, const bf16* kc_hi,
                const bf16* kc_lo, const uint8_t* kpm, int M, const int* key_len, const int* page_mw, int ks,
                float* partial, int* counters, const int* tpos, int t0, int L, float* out);
void add_i32(Ctx* c, int* p, int v);
void build_inst_prompts(Ctx* c, const int* pt_tokens, int pt_stride, int n_prompt, const int* ntok, int B, int Ncap,
                        int sos, int* tokens, int tstride);
void fill_i32(Ctx* c, int* p, long n, int v);
// Window readings of dense pages (dense.cu; rule: dense_core.h): sequence q of S (window q % P of grid (nx, ny), tokens
// tok [S][tstride] with n_prompt prompt tokens, ntok / finished of the point loop) -> its owned points xy [S][max_pts][2]
// and out [S][2] = (count, saturated).  One launch.
void dense_own(Ctx* c, int S, int P, const int* tok, int tstride, int n_prompt, const int* ntok, const int* finished,
               int nb, int nx, int ny, int max_pts, int* xy, int* out);

}  // namespace alm
