/*
 * libalm_ocr.so -- C-ABI of the H100-native (sm_90a) OCR forward path.
 *
 * The reference (AlibabaResearch/AdvancedLiterateMachinery) has no FFI table; its boundary for this
 * path is two Python `nn.Module.forward` call sites plus two checkpoint layouts (SURVEY.md 8b):
 *
 *   OmniParser : `output = model(samples, seqs)`      OCR/OmniParser/engine/val.py:35
 *                (OmniParser.forward, OCR/OmniParser/model/omniparser.py:19-32)
 *   MGP-STR    : `model(image, is_eval=True)`         OCR/MGP-STR/demo.py:33, test_final.py:140
 *                (MGPSTR.forward, OCR/MGP-STR/modules/mgp_str.py:96-101)
 *   weights    : torch.load(path)['model']            OCR/OmniParser/utils/checkpointer.py:20,44-47
 *                bare state_dict 'module.mgp_str.*'   OCR/MGP-STR/test_final.py:348,356
 *
 * The only native-API precedent in the reference is the two-function iOS library
 * `init_ocr(path, threads)` / `ocr_recognize(data, w, h, c, flag)`
 * (OCR/LiteWeightOCR/.../Headers/LiteWeight_Mobile_OCR_Recognize.h:17-19); this header keeps that
 * shape: init -> load -> run -> free, plain pointers and sizes, no C++ or torch types.
 *
 * Conventions: every function returns 0 or a negative ALM_ERR_* code and never throws across the
 * ABI; `alm_last_error` gives the message.  One `alm_ctx` per GPU per thread (no internal locking).
 * All kernels are enqueued on the context's stream.  Inputs are caller-owned (host or device
 * pointers are both accepted: host buffers are staged through pinned memory inside the call);
 * outputs are written to caller-provided host buffers after a stream synchronise.
 */
#ifndef ALM_OCR_H_
#define ALM_OCR_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define ALM_API __attribute__((visibility("default")))
#else
#define ALM_API
#endif

#define ALM_OK 0
#define ALM_ERR_INVALID (-1)   /* bad argument / missing tensor / shape mismatch          */
#define ALM_ERR_CUDA (-2)      /* CUDA runtime or driver error (message has the call)      */
#define ALM_ERR_OOM (-3)       /* workspace arena or weight slab exhausted                 */
#define ALM_ERR_STATE (-4)     /* call order violated (e.g. decode before encode)          */
#define ALM_ERR_UNSUPPORTED (-5)

typedef struct alm_ctx alm_ctx;

/* model kinds for alm_load_weights */
#define ALM_MODEL_OMNI_SPOT 1 /* OmniParser text spotting (V = 1104)                         */
#define ALM_MODEL_OMNI_KIE 2  /* OmniParser KIE: V = 1104 + vie_categories (derived from V) */
#define ALM_MODEL_MGPSTR 3    /* MGP-STR (dim/depth/heads derived from the tensors)          */

/* element types of alm_tensor_desc.data */
#define ALM_F32 0
#define ALM_F16 1
#define ALM_BF16 2
#define ALM_I64 3

/* One state-dict entry.  `name` is the reference key verbatim
 * (e.g. "backbone.0.layers.2.blocks.5.attn.qkv.weight", "module.mgp_str.blocks.0.norm1.bias").
 * `data` is a HOST pointer (or NULL: shape-only placeholder, see alm_load_weights); the library converts and uploads,
 * the caller keeps ownership. */
typedef struct alm_tensor_desc {
  const char* name;
  const void* data;
  int dtype;
  int ndim;
  int64_t shape[4];
} alm_tensor_desc;

/* ---- lifecycle ---------------------------------------------------------------------------- */
/* device: CUDA ordinal.  stream: a cudaStream_t to enqueue on, or NULL for a private stream. */
ALM_API int alm_init(int device, void* stream, alm_ctx** out);
ALM_API void alm_free(alm_ctx* ctx);
ALM_API const char* alm_last_error(const alm_ctx* ctx); /* valid until the next call on ctx */
ALM_API const char* alm_version(void);

/* options: "nsplit" (3 = bf16x3 split operands, fp32-class results [default]; 1 = single-pass bf16),
 *          "gemm_impl" (0 = wgmma [default], 1 = SIMT debug kernel), "workspace_mb", "profile_gemm",
 *          "trace_gemm" (capacity; see alm_trace_read),
 *          "fuse_ln_gemv" (point loop: 1 = every pre-LayerNorm runs inside the GEMV that consumes it, 13 fewer dependent
 *          launches per token [default]; 0 = separate LayerNorm launches),
 *          "kv_decoders" (3 = alm_omni_encode fills the cross-attention K/V caches of the pt, poly and rec decoders
 *          [default]; 1 = only the point decoder's, for callers that run alm_omni_decode_points alone),
 *          "attn_impl" (ViT attention of MGP-STR: 0 = fused flash-style mma.sync kernel, scores / probabilities never
 *          leave registers [default]; 1 = score GEMM + softmax + P.V GEMM, the A/B reference),
 *          "wattn_impl" (0 = mma.sync window attention, one CTA per (window, head), 1 = fp32 SIMT debug kernel, 3 = persistent
 *          mma.sync kernel fed by a TMA + mbarrier ring, one head pair per 128-byte row segment, bias in shared memory [default]),
 *          "small_grid_cap" (0 = off [default]; n = small GEMM launches use at most n CTAs so that concurrent
 *          streams / in-flight batches can share the GPU),
 *          "decode_streams" (polygon and recognition loops that do not run as one joint pass -- recognition beams,
 *          <= 32 single-instance sequences, xattn_impl 1, joint_decode 0 -- 2 = overlap on two streams [default], 1 = serial),
 *          "use_graphs" (1 = replay captured CUDA graphs for the per-token decode steps [default], 0 = eager),
 *          "joint_decode" (1 = the polygon and recognition loops run as one joint pass where they can [default];
 *          0 = every decode runs them as two single-decoder loops, as decode_streams selects -- the A/B reference),
 *          "xattn_impl" (0 = fused flash-style decoder cross-attention [default]; 1 = unfused score GEMM + softmax +
 *          P.V GEMM / fp32 single-query kernel, the A/B reference -- must be set before alm_omni_encode; 2 = the mma.sync
 *          kernel with a TMA + mbarrier operand ring),
 *          "xattn_ctas_per_sm" (persistent grid of the fused cross-attention: 1..3 CTAs per SM, default 2),
 *          "sattn_wide" (1 = CTA per (sequence, head) self-attention step when few sequences are live [default]),
 *          "enc_grid_cap" / "dec_grid_cap" (0 = off [default]; n = GEMM launches of alm_omni_encode / of the decode
 *          loops use at most n CTAs), "decode_priority" (1 = decode loops run on internal high-priority streams;
 *          default 0) -- co-scheduling knobs for several contexts on one GPU,
 *          "debug_skip" (timing experiments only: bit mask of decoder-layer kernel classes NOT launched; results
 *          are garbage; default 0). */
ALM_API int alm_set_option(alm_ctx* ctx, const char* key, long value);
/* block until everything enqueued on the context's stream has finished */
ALM_API int alm_synchronize(alm_ctx* ctx);
/* kernels launched on this context since the last call with reset != 0 */
ALM_API long alm_launch_count(alm_ctx* ctx, int reset);

/* Per-GEMM device timing (measurement aid, off by default): after alm_set_option(ctx, "profile_gemm", 1) every
 * tensor-core GEMM launch is bracketed by CUDA events on the context stream.  alm_profile_read synchronises,
 * returns the summed kernel time (ms), the summed algorithmic FLOPs (2*M*N*K) and the launch count, and clears. */
ALM_API int alm_profile_read(alm_ctx* ctx, double* gemm_ms, double* gemm_flops, long* gemm_launches);
/* In-kernel GEMM timeline (measurement aid): after alm_set_option(ctx, "trace_gemm", capacity) CTA 0 of every
 * wgmma GEMM stamps %globaltimer at entry and exit.  Records are 6 x u64: start ns, end ns, M, N, K,
 * tiles*1000 + BLOCK_N.  Works inside graph replays.  Reading clears the buffer. */
ALM_API int alm_trace_read(alm_ctx* ctx, unsigned long long* out, int max_records, int* n_records);
/* Times `iters` back-to-back launches of one [M,K]x[N,K]^T GEMM (operands pre-split, resident) with CUDA events
 * on the context stream; ms_per_launch is the average kernel duration. */
ALM_API int alm_bench_gemm(alm_ctx* ctx, int M, int N, int K, int iters, float* ms_per_launch);
/* Replay cost (microseconds per node) of a captured chain of `nodes` trivial dependent kernels. */
ALM_API int alm_bench_graph_floor(alm_ctx* ctx, int nodes, int iters, float* us_per_node);
/* Same, batched, with a choice of epilogue (split_out: bf16 hi/lo output; act: 0/1/2).  detail_out is reserved and must
 * be NULL (the GEMM records no per-role stamps). */
ALM_API int alm_bench_gemm_ex(alm_ctx* ctx, int M, int N, int K, int batch, int split_out, int act, int iters,
                              float* ms_per_launch, unsigned long long* detail_out);

/* Replaces reference `model.load_state_dict(torch.load(path)['model'])`
 * (OCR/OmniParser/utils/checkpointer.py:44-47; OCR/MGP-STR/test_final.py:353-356). */
ALM_API int alm_load_weights(alm_ctx* ctx, int model_kind, const alm_tensor_desc* tensors, int n);
/* A descriptor with data == NULL is a shape-only placeholder: the tensor is laid out (zeros) exactly as if it had been
 * loaded, and its values arrive later through alm_broadcast_weights -- what the non-root ranks of a multi-GPU job do. */

/* One model, many execution contexts: `ctx` (same device as `owner`) serves the weights already resident in `owner`
 * -- no copy, the device slabs are reference-counted and freed with the last context using them.  Per-batch state
 * (arena, K/V caches, captured graphs, stream) stays private to each context, so contexts can run concurrently from
 * different host threads.  Replaces the reference's one-module-per-process shape (OCR/OmniParser/model/__init__.py:7-19)
 * for serving several batches in flight per GPU. */
ALM_API int alm_share_weights(alm_ctx* ctx, alm_ctx* owner);

/* Stream ordering for device-resident inputs / outputs.  The context enqueues on its own stream (alm_init), which is
 * NOT ordered with the caller's streams: before passing device buffers written on `producer_stream` call
 * alm_stream_wait (the context's stream waits for everything enqueued on producer_stream so far); before reading
 * device outputs (alm_pre_*) on `consumer_stream` call alm_stream_release.  Host buffers need neither. */
ALM_API int alm_stream_wait(alm_ctx* ctx, void* producer_stream /* cudaStream_t */);
ALM_API int alm_stream_release(alm_ctx* ctx, void* consumer_stream /* cudaStream_t */);

/* ---- multi-GPU (SURVEY.md 8b/8e): pages shard across GPUs with no data-path collective ------- */
/* The reference has no inference collective (its NCCL use is DDP training, OCR/OmniParser/utils/dist.py:25,43-44);
 * a data-parallel serving job needs two: ONE broadcast of the weights at start-up and ONE gather of the decoded
 * sequences per batch.  NCCL is bound at run time (dlopen libnccl.so.2); ALM_ERR_UNSUPPORTED if it is absent.
 *   rank 0: alm_comm_unique_id(id) -> ship the 128 bytes to the other ranks by any means (file, socket, MPI, ...)
 *   all   : alm_comm_init(ctx, id, rank, world)        (or alm_comm_attach with a communicator the caller owns)
 *   all   : alm_load_weights (root: real tensors; others: shape-only placeholders), then alm_broadcast_weights(ctx, 0):
 *           the converted bf16 hi/lo planes and fp32 vectors travel once over NVLink straight into place
 *   batch : alm_gather_sequences(ctx, buf, bytes, recv): all-gather of one fixed-size packed buffer per rank
 *           (send: host or device; recv: host, world * bytes, rank-major, or NULL), on the context's stream.
 * With world == 1 (no communicator) broadcast is a no-op and gather a copy.
 * Several contexts of one process (each with its own communicator) must issue their collectives in ONE order that is the
 * same on every rank -- NCCL's rule for multiple communicators: a gather kernel spins on the device until its peers arrive,
 * and two ranks that start different contexts' gathers first can block each other for good.  Number the batches the same
 * way on every rank and issue gather(batch s) only after gather(batch s - 1) returned (dist.CollectiveOrder in the Python
 * adapter; a mutex + counter in a C host). */
ALM_API int alm_comm_unique_id(void* id128);
ALM_API int alm_comm_init(alm_ctx* ctx, const void* id128, int rank, int world);
ALM_API int alm_comm_attach(alm_ctx* ctx, void* nccl_comm /* ncclComm_t, caller-owned */, int rank, int world);
ALM_API int alm_broadcast_weights(alm_ctx* ctx, int root);
ALM_API int alm_gather_sequences(alm_ctx* ctx, const void* send, size_t bytes_per_rank, void* recv_host);

/* ---- OmniParser ---------------------------------------------------------------------------- */
/* Vocabulary / decode configuration: OCR/OmniParser/utils/parser.py:16-21,91-103. */
typedef struct alm_decode_cfg {
  int num_bins;       /* 1000 */
  int pt_eos, poly_eos, rec_eos, pt_sos, poly_sos, rec_sos, recog_pad;
  int pt_seq_length;  /* --pt_seq_length : max generated pt tokens                           */
  int rec_length;     /* --rec_length    : 25                                                */
  int poly_length;    /* 32 (transformer.py:254)                                             */
  int vie_categories; /* 0 for text spotting                                                 */
  int max_instances;  /* capacity of the per-image output buffers (>= pt_seq_length / 2)      */
} alm_decode_cfg;

/* Replaces `features, pos = self.backbone(samples)`, FPN and input_proj
 * (OCR/OmniParser/model/omniparser.py:20-31): Swin-B encoder -> FPN -> 1x1 stride-2 projection.
 * img  : f32 [B,3,H,W] normalised pixels (NestedTensor.tensors), host or device.
 * mask : u8  [B,H,W], 1 = padding (NestedTensor.mask), host or device, or NULL for all-valid.
 * The image memory ([B, M, 512], M = ceil(H/16)*ceil(W/16)) stays resident in the context. */
ALM_API int alm_omni_encode(alm_ctx* ctx, const float* img, const uint8_t* mask, int B, int H, int W);

/* Staged-parity readbacks (host buffers).
 * level 0..3 : LN'd Swin stage outputs, NHWC f32 [B, S_l, S_l', 128<<l]  (joiner.py:10-18)
 * which 0 = memory [B,M,512], 1 = sine position embedding [B,M,512]       (position_embedding.py:24-44) */
ALM_API int alm_omni_get_feature(alm_ctx* ctx, int level, float* out, size_t out_elems);
ALM_API int alm_omni_get_memory(alm_ctx* ctx, int which, float* out, size_t out_elems);
ALM_API int alm_omni_memory_shape(alm_ctx* ctx, int* B, int* h, int* w);

/* Pages of different sizes in one batch, each with the reference's batch-1 result: page b is encoded as the reference
 * encodes `nested_tensor_from_tensor_list([page_b])` -- its own grid, no mask, its own sine position embedding.
 * img : f32 [B,3,Hc,Wc] (the NestedTensor layout of alm_pre_omni_pages), host or device; page b is the top-left
 *       heights[b] x widths[b] of slot b, and no pixel outside that rectangle is read.  heights / widths: host [B].
 * The pages of one size are encoded together; each page's memory grid is reported by alm_omni_page_shapes.  When the
 * sizes differ:
 *   alm_omni_get_memory returns [B, Mmax, 512], Mmax = max_b mh_b * mw_b: page b's rows first (row-major over its own
 *   grid), zeros after them; alm_omni_memory_shape returns ALM_ERR_STATE and alm_omni_get_feature ALM_ERR_UNSUPPORTED.
 *   Every decode entry serves the batch, each page decoded as in a batch-1 call, and the cross-attention streams only
 *   each page's own keys.
 * When all pages have one size the state is that of alm_omni_encode(cropped pages, NULL, B, h, w).
 * Errors: ALM_ERR_INVALID for B < 1 or a page under 32 x 32 or larger than the canvas; ALM_ERR_STATE before the weights
 * are loaded; ALM_ERR_OOM as alm_omni_encode. */
ALM_API int alm_omni_encode_pages(alm_ctx* ctx, const float* img, int B, int Hc, int Wc, const int* heights,
                                  const int* widths);
/* Memory grid (mh[b], mw[b]) of every page of the last alm_omni_encode or alm_omni_encode_pages (host [B] each). */
ALM_API int alm_omni_page_shapes(alm_ctx* ctx, int* mh, int* mw);

/* Replaces `self.transformer(self.input_proj(src), mask, pos, sequence)` in eval mode
 * (OCR/OmniParser/model/transformer.py:234-286): greedy point / polygon / recognition decoding for
 * every encoded image, each image keeping the reference's batch-1 semantics.
 * pt_prompt: int64 [n_prompt] (engine/val.py:25-28).  Outputs (host), per image b:
 *   n_inst[b]                         number of decoded points (0 <=> the reference returns None)
 *   pt  [b, max_inst, 2]   int64      transformer.py:134-141
 *   poly[b, max_inst, 32]  int64      transformer.py:265
 *   rec [b, max_inst, rec_length]     transformer.py:284
 *   rec_prob [b, max_inst, rec_length] f32   transformer.py:286 */
ALM_API int alm_omni_decode(alm_ctx* ctx, const int64_t* pt_prompt, int n_prompt, const alm_decode_cfg* cfg, int32_t* n_inst,
                    int64_t* pt, int64_t* poly, int64_t* rec, float* rec_prob);

/* Reading at caller points: the polygon and recognition loops of the encoded batch (transformer.py:249-284) with the
 * point loop (decode_pt_seq, :102-141) replaced by the caller's points -- each instance is decoded from [x, y, sos]
 * alone, so a point names the word to read (training prompts them with each word's centre, dataset/collate_fn.py:
 * 117-138).  xy int32 [B][cap][2] = (x, y) in bins, 0 <= v < num_bins; count int32 [B], 0 <= count[b] <=
 * min(cap, max_instances).  Page b's rows are its count[b] points in the given order, no dedupe: the rows
 * alm_omni_decode runs for its own points, so points taken from a decode reproduce its poly / rec / rec_prob and lists
 * bit for bit.  Outputs (host) in alm_omni_decode's layout with max_inst = cap: poly int64 [B][cap][32], rec int64
 * [B][cap][rec_length], rec_prob f32 [B][cap][rec_length]; rows past count[b] are 0.  Recognition candidates, beams and
 * character locations apply as in alm_omni_decode (same combination rules), read back in the layout [B][cap]...
 * Works on batches of alm_omni_encode (with or without mask) and alm_omni_encode_pages.  The point-loop phase of
 * alm_omni_last_timing is 0.
 * Errors, before any device work and leaving the context usable: ALM_ERR_INVALID for a bin outside [0, num_bins), a
 * count outside [0, min(cap, max_instances)], cap < 1, poly_length != 32, rec_length outside 1..1021, vie_categories
 * other than the checkpoint's or a KIE checkpoint (KIE classes come from the point loop); ALM_ERR_STATE before
 * alm_omni_encode or when the batch was encoded with kv_decoders < 3. */
ALM_API int alm_omni_decode_at(alm_ctx* ctx, const int32_t* xy, const int32_t* count, int cap, const alm_decode_cfg* cfg,
                               int64_t* poly, int64_t* rec, float* rec_prob);

/* Several window prompts per image in one pass: for image b and prompt p the result equals the reference's batch-1 call
 * `model(image_b, [prompt_{b,p}, poly_sos, rec_sos, size])`.  A prompt is [x0, y0, x1, y1, c_lo, c_hi, pt_sos] (box in
 * coordinate bins, character range offset by num_bins; dataset/collate_fn.py:46-115) or the 5-token form without the
 * character range.  The B * P point sequences share one pass over each image's cross-attention K/V per token; the
 * polygon and recognition loops run once per distinct (x, y) of an image and their results are copied to every
 * (image, prompt) slot that holds the point.
 * prompts int64 [B][P][n_prompt] (1 <= P <= 16, 1 <= n_prompt <= 16, every token in [0, V)); outputs per (image, prompt)
 * slot, the layout of alm_omni_decode with B * P images:
 *   n_inst [B][P]; pt [B][P][max_inst][2]; poly [B][P][max_inst][32]; rec, rec_prob [B][P][max_inst][rec_length].
 * Errors: ALM_ERR_INVALID for P, n_prompt or a token out of range, a KIE checkpoint, max_instances < pt_seq_length / 2;
 * ALM_ERR_STATE before alm_omni_encode or when the batch was encoded with kv_decoders < 3; ALM_ERR_OOM when the
 * point loop's self-attention caches (16 MB per sequence at a full 1024-step table) do not fit the workspace. */
ALM_API int alm_omni_decode_prompts(alm_ctx* ctx, const int64_t* prompts, int P, int n_prompt, const alm_decode_cfg* cfg,
                                    int32_t* n_inst, int64_t* pt, int64_t* poly, int64_t* rec, float* rec_prob);

/* Dense pages: text spotting of pages with more words than one point sequence holds (two tokens per word, at most
 * pt_steps = min(pt_seq_length, 1025 - n_prompt) steps), read in the spatial windows the model was trained on
 * (DESIGN 4.16; the rule in full is in dense_core.h).
 *   saturation  a point sequence is saturated when it runs all pt_steps steps without choosing pt_eos; its points are
 *               kept as alm_omni_decode keeps them (trailing odd token dropped).
 *   windows     on an axis cut into n: inter = min(int(num_bins / n), num_bins - 1), window i spans
 *               [i inter, min(i inter + inter, num_bins - 1)] (dataset/collate_fn.py:46-83).  Grid (nx, ny), nx, ny in
 *               1..3; window w = iy nx + ix (top to bottom, then left to right).  Its prompt is pt_prompt with tokens
 *               0..3 replaced by the window's box; pt_prompt's box must be (0, 0, num_bins - 1, num_bins - 1).
 *   ownership   (x, y) belongs to window (sx, sy, ex, ey) iff sx < x <= ex or sx = 0 <= x <= ex, and the same in y, so
 *               the windows partition the page.  A window reading keeps only the points it owns, on the device, before
 *               the polygon and recognition loops.
 *   levels      (nx, ny) = (0, 0), 'auto': every page is read with pt_prompt; a page that does not saturate keeps that
 *               reading (grid (1, 1)).  A saturated page is read at 2 x 2; if any of its windows saturates it is read at
 *               3 x 3 instead.  A 3 x 3 window that still saturates keeps its points and is flagged.  An explicit grid
 *               reads every page once at that grid.  When no page saturates, 'auto' is alm_omni_decode: the same
 *               launches and outputs.
 *   merge       a page read in windows is merged by alm_omni_merge_readings' rule over its windows (box of the 16
 *               vertices in bins, decode_pred_seq's score, IoU >= iou): a row is dropped iff a row of another window of
 *               the page overlaps it and ranks above it.
 * Only the saturated pages are read again, as runs of consecutive pages of the encoded batch: a page that is done adds
 * no query rows and its cross-attention K/V are not streamed.  The polygon and recognition loops run over every kept
 * point of every page in passes of at most B x max_instances rows, so the workspace peak is alm_omni_decode's.
 * Outputs (host), per page b at cap rows: n_inst [B]; pt [B][cap][2], poly [B][cap][32], rec / rec_prob
 * [B][cap][rec_length] in alm_omni_decode's layout, each page's kept rows in (window, instance) order; window int32
 * [B][cap]; grid int32 [B][2] = (nx, ny) used; saturated uint8 [B][9] per window of that grid (0 past its windows).
 * Errors, before any device work and leaving the context usable: ALM_ERR_INVALID for a KIE checkpoint, a grid
 * outside the trained set, n_prompt outside 5..16 or a token out of range, a box other than the whole page, iou
 * outside (0, 1] or not finite, recognition candidates / beams / character locations switched on, max_instances <
 * pt_seq_length / 2, or cap below what the grid can produce (its window count, 9 for 'auto', x pt_steps / 2);
 * ALM_ERR_STATE before alm_omni_encode or when the batch was encoded with kv_decoders < 3. */
ALM_API int alm_omni_decode_dense(alm_ctx* ctx, const int64_t* pt_prompt, int n_prompt, const alm_decode_cfg* cfg,
                                  int nx, int ny, double iou, int cap, int32_t* n_inst, int64_t* pt, int64_t* poly,
                                  int64_t* rec, float* rec_prob, int32_t* window, int32_t* grid, uint8_t* saturated);

/* The loops the last alm_omni_decode_dense ran beyond its level-0 decode, in order: out int32 [n_loops][4] = (kind,
 * img0, nimg, per_page) over pages img0 .. img0 + nimg - 1 of the encoded batch; kind 0 is a window point loop with
 * per_page = nx ny window prompts, kind 1 a polygon / recognition pass with per_page rows per page.  None when no page
 * saturated.  elems = capacity of out (4 per loop); out NULL with elems 0 reports n_loops alone.  ALM_ERR_INVALID for a
 * null n_loops, or out NULL or too small otherwise. */
ALM_API int alm_omni_get_dense_loops(alm_ctx* ctx, int32_t* out, size_t elems, int32_t* n_loops);

/* The point loop alone: `decode_pt_seq` (transformer.py:102-141) for every encoded image -- the structure / layout
 * sequence decoders built on this model (the unreleased table-recognition head, OCR/OmniParser/README.md:85-101) run
 * exactly this loop for hundreds of tokens.  Outputs (host), per image b: n_tok[b] generated tokens (prompt stripped,
 * a trailing odd token dropped as in :138-139), pt_tokens[b, pt_seq_length] int64, pt_probs[b, pt_seq_length] f32
 * (may be NULL).  max_instances / poly_length of cfg are ignored. */
ALM_API int alm_omni_decode_points(alm_ctx* ctx, const int64_t* pt_prompt, int n_prompt, const alm_decode_cfg* cfg,
                                   int32_t* n_tok, int64_t* pt_tokens, float* pt_probs);

/* KIE variant (--infer_vie): replaces the eval branch with `decode_vie_pt_poly_rec_seq` (transformer.py:143-217,243-246).
 * The pt loop emits (x, y, class) triples (:117-123) with the class slot restricted to the last vie_categories
 * ids; every (x, y) pair found by the reference's walk (:148-210) gets a polygon and a transcription whose
 * softmax runs over the first V - vie_categories logits (:156,176).  Outputs (host), per image b:
 *   n_tok[b]; pt_tokens[b, pt_seq_length] int64 and pt_probs[b, pt_seq_length] f32 (prompt stripped, :132-141);
 *   n_inst[b]; inst_pos[b, max_inst] = index in pt_tokens where the pair starts;
 *   poly[b, max_inst, 32], rec[b, max_inst, rec_length], rec_prob[b, max_inst, rec_length].
 * The entity grouping / class names / rectangles (:163-169,190-215) are plain host post-processing over these. */
ALM_API int alm_omni_decode_kie(alm_ctx* ctx, const int64_t* pt_prompt, int n_prompt, const alm_decode_cfg* cfg,
                                int32_t* n_tok, int64_t* pt_tokens, float* pt_probs, int32_t* n_inst, int32_t* inst_pos,
                                int64_t* poly, int64_t* rec, float* rec_prob);

/* Recognition candidates: the k most likely characters at every step of the recognition loop, for lexicon matching,
 * dictionary correction or routing uncertain words to review.  k (ALM_MAX_CANDIDATES at most) applies to the following
 * alm_omni_decode / alm_omni_decode_prompts / alm_omni_decode_kie calls of the context; 0 (the default) records none and
 * leaves every output, launch and captured graph as it is without this call.
 * At each of the rec_length steps along the greedy path the candidates are the k classes of the step's allowed set
 * (num_bins..recog_pad and rec_eos, the set `rec` is chosen from) with the highest softmax probability, ordered by
 * probability, lowest id first on equal probability, each with its probability under the step's softmax over
 * logits[:nsoft] (V for spotting, V - vie_categories for KIE; not renormalised over the candidates).  Candidate 0 is
 * rec / rec_prob bit for bit.  Fewer than k allowed classes: the rest are id -1, probability 0.
 * alm_omni_get_rec_candidates returns those of the last decode in the layout of rec with a trailing k:
 *   ids int64 / probs f32 [slot][max_instances][rec_length][k] (slot = image, or (image, prompt) for
 *   alm_omni_decode_prompts, where a point shared by several slots carries its candidates to each); entries of
 *   instances past n_inst are 0.  elems = capacity of each buffer, in elements.
 * Errors: ALM_ERR_INVALID for k outside 0..ALM_MAX_CANDIDATES, null buffers or elems below the count; ALM_ERR_STATE when
 * the last of those decodes ran with k = 0 (or none ran). */
#define ALM_MAX_CANDIDATES 8
ALM_API int alm_omni_set_rec_candidates(alm_ctx* ctx, int k);
ALM_API int alm_omni_get_rec_candidates(alm_ctx* ctx, int64_t* ids, float* probs, size_t elems);

/* Recognition beam search: the n best transcriptions of every text instance, each with a sequence score that lexicon
 * matching, dictionary correction or review routing can rank.  W (ALM_MAX_BEAMS at most) and the length penalty
 * alpha in [0, 2] apply to the following alm_omni_decode / alm_omni_decode_prompts / alm_omni_decode_kie calls of the
 * context; W = 0 (the default) is the greedy loop, with every output, launch and captured graph as without this call.
 * The point and polygon loops stay greedy.  Per (slot, instance):
 *   - allowed classes: num_bins..recog_pad and rec_eos (the set rec is chosen from); p_c is the class's probability
 *     under the step's fp32 softmax over logits[:nsoft] (V for spotting, V - vie_categories for KIE).
 *   - rec_eos and recog_pad end a hypothesis (where decode_seq stops reading).
 *   - step 0 starts from the single prefix [x, y, rec_sos] with score 0; the other W - 1 slots are dead.
 *   - each step: a live hypothesis h expands to every allowed class c with p_c > 0, score s_h + log(p_c); a finished
 *     hypothesis offers itself, score unchanged.  The W best candidates survive, by score descending, ties to the
 *     lower parent slot, then to the lower class id.  Slots without a finite candidate are dead (id -1, score -inf).
 *   - after rec_length steps the W hypotheses are ranked by s / len^alpha (len = tokens up to and including the
 *     terminal token, or rec_length without one), ties to the lower slot.  Hypothesis 0 is rec / rec_prob, its
 *     per-step probability p_c of the chosen token; positions after the terminal token hold recog_pad, probability 0.
 * With W = 1 this is the greedy loop up to and including the first terminal token, ids and probabilities bit for bit.
 * alm_omni_get_rec_beams returns the last decode's n-best lists: ids int64 / probs f32 [slot][max_instances][W]
 * [rec_length] and scores f32 [slot][max_instances][W] (the raw log-probability sums s), slot = image, or (image,
 * prompt) for alm_omni_decode_prompts; entries of instances past n_inst are 0.  elems = capacity of ids and of probs,
 * in elements; scores holds elems / rec_length.
 * Errors: ALM_ERR_INVALID for W outside 0..ALM_MAX_BEAMS, alpha outside [0, 2], W > 0 while rec candidates are on (or
 * candidates while beams are on), null buffers or elems below the count; ALM_ERR_STATE when the last of those decodes
 * ran with W = 0 (or none ran). */
#define ALM_MAX_BEAMS 8
ALM_API int alm_omni_set_rec_beams(alm_ctx* ctx, int W, float length_penalty);
ALM_API int alm_omni_get_rec_beams(alm_ctx* ctx, int64_t* ids, float* probs, float* scores, size_t elems);

/* Character locations: where on the page the recognition decoder looked for each character it emitted, for
 * highlighting, redaction or aligning characters on a spotted page without a second recognition pass.  on != 0 applies
 * to the following alm_omni_decode / alm_omni_decode_prompts / alm_omni_decode_kie calls of the context; off (the
 * default) allocates and launches nothing and leaves every output and captured graph as without this call.
 * Map: for instance n and rec step j (the step that emits rec[n][j], all rec_length steps, also after the end token),
 * A_j is the cross-attention weight row of the last rec decoder layer (transformer.rec_decoder.layers[3]
 * .multihead_attn(...)[1][:, -1, :] in the reference's greedy step j) averaged over its 8 heads: per head
 * softmax((q_h / 8) K_h^T) over the page's live keys, q_h the head's slice of that layer's query projection of
 * LN2(x) + query_pos, K_h its slice of the K cache; masked keys and keys at or beyond the page's key count weigh 0.
 * Key positions: key k of a page with memory grid mh x mw is cell (r, c) = (k / mw, k % mw) of the stride-16 grid and
 * sits at its centre x = 16 c + 8, y = 16 r + 8, in edge coordinates of the encoder's input page (0 = left edge of
 * pixel 0; a convention: input_proj reads stride-8 cell (2r, 2c), whose FPN features also carry the upsampled
 * coarser levels over the whole 16-px cell).  Pages are top-left aligned on the canvas, so padded batches and
 * alm_omni_encode_pages use the same formula with each page's own mw.
 * Output per (instance, step), reduced on the device: cx, cy = sum A (x, y); sxx, sxy, syy = the central second
 * moments of A about (cx, cy), in encoder-input pixels.  Heads combine as mu = mean mu_h,
 * Sigma = mean (Sigma_h + (mu_h - mu)(mu_h - mu)^T), in a fixed order (bit-reproducible run to run).
 * Locations follow the greedy path, so they combine with rec candidates (candidate 0 is that path).
 * alm_omni_get_rec_locations returns those of the last decode: f32 [slot][max_instances][rec_length][5] (slot = image,
 * or (image, prompt) for alm_omni_decode_prompts, where a point shared by several slots carries its locations to
 * each); entries of instances past n_inst are 0.  elems = capacity of out, in elements.
 * Errors: ALM_ERR_INVALID when turned on while rec beams are on, when beams are turned on while locations are on, for a
 * null buffer or elems below the count; ALM_ERR_STATE when the last of those decodes ran with locations off (or none
 * ran). */
ALM_API int alm_omni_set_rec_locations(alm_ctx* ctx, int on);
ALM_API int alm_omni_get_rec_locations(alm_ctx* ctx, float* out, size_t elems);

/* Character sets: restrict the recognition loop to caller-given characters, per decode or per row -- an amount, a
 * date or an ID field (digits and ".,-/"), a licence plate (upper case and digits), a meter reading (digits).  The
 * choice is constrained at every step, so a wrong first character is never fed back as filtering the text afterwards
 * would leave it.  The rule:
 *   - chars are the checkpoint's characters, classes num_bins + i (n_chars = recog_pad - num_bins - 1, 95 by
 *     default).  A set is a subset of chars with at least one character: allowed uint8 [n_sets][n_chars], nonzero =
 *     chars[i] in the set.
 *   - while a set is in force, rec step j of an instance may choose num_bins + i for every chars[i] in the set, the
 *     unknown class recog_pad - 1, recog_pad and rec_eos: the allowed set of the recognition loop intersected with the
 *     caller's characters.  A word can still end, and a glyph the set cannot name can still be read as unknown, which
 *     decode_seq drops, so every character of every returned text is in the set.  The full set gives every output,
 *     launch and list bit for bit as without a set.
 *   - a chosen class keeps its probability under the step's softmax over logits[:nsoft] (not renormalised over the
 *     set), so the decode_pred_seq score of a forced word drops.  Ties go to the lower id.
 *   - candidates are the k best classes of the constrained set (id -1, probability 0 past its end; candidate 0 is
 *     rec); beams expand only into it (W = 1 is still the greedy loop up to the terminal token); character locations
 *     follow the constrained path.  The point and polygon loops are unchanged.
 * n_sets = 0 turns the setting off (the default: nothing allocated, copied or launched).  With row_set NULL (n_rows 0)
 * every instance of the following alm_omni_decode / _prompts / _kie / _at / _dense calls uses set 0.  A row_set is
 * read by alm_omni_decode_at alone: int32 [B][cap] of that call (n_rows = B cap), point n of page b reads with set
 * row_set[b cap + n].  The setting is copied and stays in force until the next call.
 * Errors: ALM_ERR_INVALID here, leaving the previous setting, for n_sets outside 0..ALM_MAX_CHARSETS, a null allowed or
 * n_chars < 1, an empty set, a set index outside [0, n_sets), or row_set and n_rows not given together; ALM_ERR_INVALID
 * from a decode, before any device work and leaving the context usable, for n_chars other than recog_pad - num_bins -
 * 1, row sets with any entry other than alm_omni_decode_at, or n_rows other than its B cap. */
#define ALM_MAX_CHARSETS 65536
ALM_API int alm_omni_set_rec_charset(alm_ctx* ctx, const uint8_t* allowed, int n_sets, int n_chars,
                                     const int32_t* row_set, size_t n_rows);

/* Teacher-forced logits: replaces `Transformer.decode(input_seq, memory, mask, pos_embed, input_type)`
 * (transformer.py:74-100) for image `image`: seq int64 [n_seq, len] -> logits f32 [n_seq, len, V].
 * kind: 0 = pt, 1 = poly, 2 = rec. */
ALM_API int alm_omni_decode_logits(alm_ctx* ctx, int image, int kind, const int64_t* seq, int n_seq, int len, float* logits);
ALM_API int alm_omni_vocab(alm_ctx* ctx);
/* Device time (CUDA events on the context stream) of the last alm_omni_encode and of the two halves of the last
 * decode: the point loop, and the polygon + recognition loops (incl. the host round trip between them); -1 = n/a. */
ALM_API int alm_omni_last_timing(alm_ctx* ctx, float* encode_ms, float* pt_ms, float* polyrec_ms);

/* ---- MGP-STR ------------------------------------------------------------------------------- */
/* Replaces `model(image, is_eval=True)` (OCR/MGP-STR/modules/mgp_str.py:96-101).
 * img: f32 [B,3,32,128] in [0,1].  Any output pointer may be NULL.  Host buffers:
 *   attn   [3][B,27,257] f32 (char, bpe, wp A^3 maps)
 *   char_logits [B,27,38], bpe_logits [B,27,50257], wp_logits [B,27,30522]  f32
 *   ids    [3][B,27] int32 top-1 ids, prob [3][B,27] f32 max softmax prob (demo.py:36-60).
 * The model variant comes from the checkpoint: tiny / small / base / large (embed 192 / 384 / 768 / 1024, 64-wide heads,
 * mgp_str.py:176-230) and the char-only CHAR-STR ablation (modules/char_str.py:43-81: one A^3 module, logits through
 * timm's `head`).  For CHAR-STR only the first plane of attn / ids / prob and char_logits are written; the class
 * counts of the heads (the widths of the logit buffers) are reported by alm_mgpstr_info. */
ALM_API int alm_mgpstr_info(alm_ctx* ctx, int* dim, int* depth, int* heads, int* n_a3, int* vocab3 /*[3]*/);
ALM_API int alm_mgpstr_forward(alm_ctx* ctx, const float* img, int B, float* attn, float* char_logits, float* bpe_logits,
                       float* wp_logits, int32_t* ids, float* prob);
/* alm_mgpstr_forward reduced to the k most likely classes per crop and position (1 <= k <= ALM_MAX_CANDIDATES), over
 * each head's whole vocabulary: ids int32 / probs f32 [3][B,27,k] host buffers, ordered by softmax probability, lowest
 * id first on equal probability.  Candidate 0 is the ids / prob of alm_mgpstr_forward bit for bit.  No logits leave the
 * device.  CHAR-STR writes the first plane only.  Errors: ALM_ERR_INVALID for k or null arguments; ALM_ERR_STATE when
 * the context holds no MGP-STR checkpoint. */
ALM_API int alm_mgpstr_topk(alm_ctx* ctx, const float* img, int B, int k, int32_t* ids, float* probs);
/* Where each recognised character is: alm_mgpstr_forward's ids / prob (alm_mgpstr_topk's when k >= 1) plus one box per
 * predicted character (char head) or sub-word token (BPE / WordPiece heads), reduced on the device from the A^3 maps
 * that the reference's demo draws over the crop (OCR/MGP-STR/demo.py:119-124).  One extra kernel launch per head; no
 * map leaves the device.  Per head and crop:
 *   - n: char head: the reference's char_pred_EOS, the string index of '[s]' in char_decode(ids[1:]) (each '[GO]'
 *     before it counts 4 characters, every other token 1), 0 without '[s]', at most 26.  This equals the string
 *     index whenever the character tokens are single characters and none of them spell '[s]' before the real one.
 *     BPE / WordPiece: the index of the first end id (2 / 102) in ids[1:], 26 without one.  CHAR-STR has the char
 *     head only.  Boxes follow the top-1 ids (candidate 0 when k >= 1).
 *   - slot j = 0..n-1 takes the map of token j + 1, patches only: attens[h][b][:, 1:].view(-1, 8, 32)[1:n+1].  In
 *     double with sums in a fixed sequential order: column masses c[x] = sum over the 8 rows, m = sum of c; each
 *     column's mass spread evenly over input pixels [4x, 4x + 4) of the 128-wide input; the box runs from the 10 % to
 *     the 90 % point of that cumulative mass and over the full crop height; the centre is the mass-weighted centroid
 *     (columns at 4x + 2, rows at 4y + 2).  A map of mass 0 gives the whole input and its middle.
 *   - input edge coordinate u -> crop pixel X = u cw / 128 - 0.5, v -> Y = v ch / 32 - 0.5 (crop size cw x ch); the
 *     box's top and bottom edges are the crop's first and last rows (Y = 0, ch - 1), which lie on the region's
 *     boundary.  Then to the page: geom_kind ALM_BOX_QUAD applies the crop -> page matrix and divides (a zero divisor
 *     gives (0, 0), where the warp samples); ALM_BOX_CURVE evaluates T(t) + (B(1 - t) - T(t)) s with t = X / (cw - 1),
 *     s = Y / (ch - 1) (0 for a side of 1); ALM_BOX_CROP stays in the 128 x 32 input's pixel coordinates.
 * geom: the exact plan each crop was cut with, n_geom == B regions: sizes int32 [B][2] (crop width, height) and geom
 * f64 [B][9] (alm_pre_quad_plan's minv) or [B][16] (alm_pre_curve_plan's ctrl); both unused (may be NULL) for
 * ALM_BOX_CROP.  n_heads must equal the checkpoint's A^3 head count (3, or 1 for CHAR-STR).  Host outputs, n_heads
 * planes each: ids / probs as alm_mgpstr_forward (k = 0) or alm_mgpstr_topk (k >= 1); n int32 [B]; boxes f32
 * [B][26][4][2] (x, y) top-left, top-right, bottom-right, bottom-left in reading direction; centres f32 [B][26][2];
 * slots >= n are zero.  Errors, before any device work: ALM_ERR_INVALID for null arguments, k outside 0..8, an unknown
 * geom_kind, n_geom != B, n_heads that does not match the checkpoint, a crop side < 1 or non-finite geometry;
 * ALM_ERR_STATE without an MGP-STR checkpoint. */
#define ALM_BOX_CROP 0
#define ALM_BOX_QUAD 1
#define ALM_BOX_CURVE 2
ALM_API int alm_mgpstr_forward_boxes(alm_ctx* ctx, const float* img, int B, int k, int geom_kind, int n_geom,
                                     const int* sizes, const double* geom, int n_heads, int32_t* ids, float* probs,
                                     int32_t* n, float* boxes, float* centres);
/* Text lines longer than MGP-STR's 32 x 128 input: the B crops are the windows alm_pre_line_crops cut from R regions
 * (windows[r] of region r, in region order; they must sum to B), and each head's tokens are stitched back into one
 * sequence per region on the device, right after the head's A^3 maps are reduced.  Region r has crop size cw x ch =
 * sizes[r] and the window layout of alm_pre_line_windows (x_i, wn).  Per head, region and window:
 *   - the window's tokens are ids positions 1 .. e - 1, e the position of the first end id in ids[1:] (char head 1
 *     '[s]', BPE 2, WordPiece 102), all 26 without one -- the BPE / WordPiece count of alm_mgpstr_forward_boxes, for
 *     the char head too ('[GO]' counts as one token here);
 *   - token j sits at X = (x_i + u wn / 128) - 0.5 on the full crop, u the centroid column of its A^3 map in the
 *     128-wide input (the rule of alm_mgpstr_forward_boxes; a map of mass 0 gives 64);
 *   - the seam between windows i and i + 1 is c_i = (x_{i+1} + x_i + wn - 1) / 2; window i keeps token j iff
 *     c_{i-1} <= X < c_i (no bound for the first / last window), so a token on a seam goes right.
 * Outputs, host, n_heads planes each: ids int32 / probs f32 [R][210]: position 0 is window 0's position 0, then the
 * kept tokens in window order and token order (n [R] of them, at most 208), then the head's end id with the last
 * window's end-token probability (0 when the last window has no end token), then the end id with probability 1.  This
 * is the layout of one crop's alm_mgpstr_forward ids / prob with T = 210, so alm_post_mgp_fuse reads it unchanged.
 * boxes f32 [R][208][4][2] / centres f32 [R][208][2]: the alm_mgpstr_forward_boxes box of every kept token with the X
 * above, mapped through the region's plan (geom f64 [R][9] minv for ALM_BOX_QUAD, [R][16] ctrl for ALM_BOX_CURVE, with
 * t = X / (cw - 1)); slots >= n are zero.  Two kernel launches per head besides the forward (box reduction and
 * stitch); only the stitched sequences leave the device.  Errors, before any device work: ALM_ERR_INVALID for null
 * arguments, R or B < 1, a kind other than quad / curve, window counts that differ from the layout of sizes or do not
 * sum to B, n_heads that does not match the checkpoint, non-finite geometry, a crop side < 1, or line buffers that do
 * not fit in the workspace; ALM_ERR_STATE without an MGP-STR checkpoint. */
ALM_API int alm_mgpstr_forward_lines(alm_ctx* ctx, const float* img, int B, int R, const int* windows, int kind,
                                     const int* sizes, const double* geom, int n_heads, int32_t* ids, float* probs,
                                     int32_t* n, float* boxes, float* centres);
/* Text that does not run upright in its crop (DESIGN 4.13): the B crops are N readings of R regions, cut by
 * alm_pre_turned_crops (lines = 1: their windows), region r's readings[r] (1 or 2) readings next to each other, reading
 * i at turns[i] (0..3 quarter-turns counter-clockwise).  Runs the forward (+ box reduction / line stitching) of all of
 * them, then keeps per region the reading with the larger fused confidence -- per head the float32 of the sequential
 * double product of its probabilities up to the end position (alm_post_mgp_fuse's rule: the char head's string index
 * of '[s]' with '[GO]' counted as 4 characters, 0 without '[s]'; BPE / WordPiece the first end id), the largest over
 * the heads -- the lower turn on equal confidence.  The choice and the gather of the kept rows are one kernel launch;
 * only R rows cross PCIe.
 *   lines 0, kind ALM_BOX_CROP (0): no boxes; N == B; ids / probs [R][27] (k = 0) or [R][27][k] per head as
 *     alm_mgpstr_forward / alm_mgpstr_topk; sizes, geom, windows, n, boxes, centres unused.
 *   lines 0, kind ALM_BOX_QUAD / ALM_BOX_CURVE: alm_mgpstr_forward_boxes' outputs of the kept readings, R rows; sizes
 *     [N][2] and geom [N][9] / [N][16] are each reading's natural (upright) plan.  Box coordinates in the turned crop
 *     go back to the upright crop by exact integer offsets before the plan maps them, so corners follow the reading.
 *   lines 1 (kind 1 / 2, k = 0): alm_mgpstr_forward_lines' outputs, R rows; windows [N] = the window count of each
 *     reading's TURNED crop (the layout of alm_pre_line_windows on the turned sides); seams and X are computed there.
 * turns_out int32 [R] and conf f32 [R] are the kept reading's turn and fused confidence.  Errors, before any device
 * work: ALM_ERR_INVALID for null arguments, a turn outside 0..3, readings other than 1 or 2 per region or not summing
 * to N, N != B without lines, window counts that disagree with the turned layout or do not sum to B, and everything
 * alm_mgpstr_forward_boxes / alm_mgpstr_forward_lines reject; ALM_ERR_STATE without an MGP-STR checkpoint. */
ALM_API int alm_mgpstr_forward_oriented(alm_ctx* ctx, const float* img, int B, int N, const int32_t* turns, int R,
                                        const int* readings, int k, int lines, int kind, const int* windows,
                                        const int* sizes, const double* geom, int n_heads, int32_t* ids, float* probs,
                                        int32_t* n, float* boxes, float* centres, int32_t* turns_out, float* conf);

/* ---- low-level ops (unit parity tests call these through the ABI; device pointers only) ------ */
/* C[M,N] f32 = A[M,K] f32 * W[N,K]^T f32 (+bias[N]) with act 0 none / 1 gelu(erf) / 2 relu; runs the same
 * operand split + wgmma kernel as the model graphs.  batch > 1: contiguous batches of A, W and C. */
ALM_API int alm_op_linear(alm_ctx* ctx, const float* A, const float* W, const float* bias, float* C, int M, int N, int K,
                  int act, int batch);
/* The same GEMM with every feature of its fused epilogue, under the context's nsplit.  A f32 [batch, M, K] and
 * W f32 [w_batch, N, K] (w_batch 1: W is shared by every batch) are split internally as in alm_op_linear; K % 4 == 0.
 * For batch b, row m and column n < N:
 *   x = act(alpha * (A_b W_b^T)[m, n] + bias_b[n or m]) + resid[b * rbs0 + rrow * ldr + n]
 *   orow = out_map ? out_map[m] : m  (negative: row m is not written),  rrow = resid_map ? resid_map[m] : orow
 *   written at b * obs0 + orow * ldo + cn, cn = col_group ? (n / col_group) * col_group_stride + n % col_group : n,
 * to out_f32 and / or the bf16 pair out_hi = bf16_rn(x), out_lo = bf16_rn(x - out_hi) (uint16 buffers; out_lo may be
 * NULL).  bias_mode 0 none / 1 per column (bias_b = bias + b * bias_bs0) / 2 per row; act 0 none / 1 gelu(erf) / 2 relu.
 * Nothing else is written.  ALM_ERR_INVALID for combinations the engine does not run: no output, row maps with
 * batch > 1, col_group with a residual or with col_group % 4 != 0 or col_group_stride % 8 != 0. */
ALM_API int alm_op_gemm(alm_ctx* ctx, const float* A, const float* W, int M, int N, int K, int batch, int w_batch,
                        float* out_f32, void* out_hi, void* out_lo, long ldo, long obs0, const float* bias, int bias_mode,
                        long bias_bs0, float alpha, int act, const float* resid, long ldr, long rbs0,
                        const int* resid_map, const int* out_map, int col_group, long col_group_stride);
/* One K-major operand of the GEMM engine as it is handed to the kernel: device bf16 hi / lo planes (uint16 elements).
 * Row r of batch (b0, b1) starts at hi + b0 * bs0 + b1 * bs1 + r * ld; only its first K elements are read (the
 * rest of the row, and anything between rows and batches, may hold anything).  nb0 / nb1 equal the problem's batch
 * extent, or 1 to broadcast the operand along that dimension (its stride is then unused).  ld, bs0, bs1 and the
 * distance lo - hi are multiples of 8 elements; lo lies after hi (the planes may be any distance apart) and may be
 * NULL when the context runs nsplit 1. */
typedef struct alm_gemm_operand {
  const void* hi;
  const void* lo;
  int rows, K;
  long ld;
  int nb0, nb1;
  long bs0, bs1;
} alm_gemm_operand;
/* The GEMM's fused epilogue with every stride the engine takes: alm_op_gemm's arguments plus obs1 (output) and rbs1
 * (residual), the strides along the second batch dimension.  Element (b0, b1, m, n) of the product is written at
 * b0 * obs0 + b1 * obs1 + orow * ldo + cn, its column bias is bias[b0 * bias_bs0 + n] (row bias: [b0 * bias_bs0 + m])
 * and its residual resid[b0 * rbs0 + b1 * rbs1 + rrow * ldr + n]; the rest as in alm_op_gemm. */
typedef struct alm_gemm_epilogue {
  float* out_f32;
  void* out_hi;
  void* out_lo;
  long ldo, obs0, obs1;
  int col_group;
  long col_group_stride;
  const float* bias;
  int bias_mode;
  long bias_bs0;
  const float* resid;
  long ldr, rbs0, rbs1;
  const int* out_map;
  const int* resid_map;
  int act;
  float alpha;
} alm_gemm_epilogue;
/* D = A B^T on operands exactly as given (no split, no copies): the engine's own entry, under the context's nsplit
 * and gemm_impl.  At nsplit 3 each k-step forms hi*hi + lo*hi + hi*lo; at nsplit 1 only hi*hi, and no lo plane is
 * read.  ALM_ERR_INVALID, before any device work, for null or host pointers, planes that are not 16-byte aligned,
 * ld / bs0 / bs1 / plane distance not a multiple of 8, lo not after hi, ld < K, batch extents that neither match nor
 * broadcast, and everything alm_op_gemm rejects. */
ALM_API int alm_op_gemm_planes(alm_ctx* ctx, const alm_gemm_operand* A, const alm_gemm_operand* B,
                               const alm_gemm_epilogue* epi);
/* softmax((q k^T) * 64^-0.5) v for B sequences of T <= 272 tokens and H heads of width 64: qkv f32 [B*T, 3*H*64] (q | k | v
 * column blocks, head h at columns h*64 of its block: the layout of timm's packed qkv Linear), out f32 [B*T, H*64].
 * Runs the fused attention kernel of the ViT blocks (scores and probabilities stay on chip). */
ALM_API int alm_op_attention(alm_ctx* ctx, const float* qkv, float* out, int B, int T, int H);
/* The same kernel on the operands the ViT blocks hand it, under the context's nsplit: qkv as device bf16 planes qkv_hi /
 * qkv_lo (uint16 buffers), row r of the B*T token rows at r * ld (ld >= 3*H*64 and a multiple of 8; only its first
 * 3*H*64 elements are read).  nsplit 3 forms q k^T and P v from hi*hi + lo*hi + hi*lo; nsplit 1 reads only the hi plane
 * (qkv_lo may be NULL).  Outputs, row stride ldo (>= H*64, a multiple of 8), each nullable: out_f32 and / or the bf16 pair
 * out_hi = bf16_rn(x), out_lo = bf16_rn(x - out_hi) (out_f32 or out_hi required; out_lo needs out_hi; out_lo is not
 * written at nsplit 1).  Columns H*64 .. ldo-1 are not written.  Every pointer is device memory aligned to 16 bytes.
 * ALM_ERR_INVALID for null or host pointers, misalignment, ld or ldo out of range, no output, or no lo plane at
 * nsplit 3; ALM_ERR_UNSUPPORTED for T > 272. */
ALM_API int alm_op_attention_ex(alm_ctx* ctx, const void* qkv_hi, const void* qkv_lo, long ld, int B, int T, int H,
                                float* out_f32, void* out_hi, void* out_lo, long ldo);
/* MGP-STR's per-row selection over the first n columns of logits f32 [rows][ld] (device): order by value descending,
 * lowest id first on equal values (fp32 values compared exactly, +0 == -0).  k 0: the top-1 id and its softmax
 * probability, ids int32 / probs f32 [rows]; k 1..8: the k best candidates, [rows][k], with the probability of every id
 * whose value equals the maximum exactly that of candidate 0, id -1 and probability 0 past the n classes.  Candidate 0
 * is the k 0 result bit for bit.  Columns n .. ld-1 are not read.  ALM_ERR_INVALID for null or host pointers, rows < 1,
 * n < 1, n > ld or k outside 0..8. */
ALM_API int alm_op_row_select(alm_ctx* ctx, const float* logits, long ld, int rows, int n, int k, int32_t* ids,
                              float* probs);
ALM_API int alm_op_layernorm(alm_ctx* ctx, const float* x, const float* gamma, const float* beta, float eps, float* y,
                     long rows, int C);
/* Swin W-MSA core on an already windowed qkv tensor [B*nWh*nWw*49, 3C] (swin_transformer.py:127-148). */
ALM_API int alm_op_window_attention(alm_ctx* ctx, const float* qkv, const float* bias_table /*[169,heads]*/, float* out,
                            int B, int nWh, int nWw, int C, int heads, int shift);
/* alm_op_window_attention with every output form of the kernels: out_f32 f32 and / or the bf16 pair out_hi =
 * bf16_rn(x), out_lo = bf16_rn(x - out_hi) (uint16 buffers), each [B*nWh*nWw*49, C] and nullable (out_f32 or out_hi
 * required; out_lo needs out_hi).  qkv f32 (q unscaled), windows in (b, window row, window column) order; the shift
 * mask (-100 between the regions of swin_transformer.py:368-387) applies for shift > 0, on the padded Hp = 7 nWh,
 * Wp = 7 nWw grid.  wattn_impl 1 runs the fp32 SIMT kernel; 0 and 3 split q * 32^-0.5, k and v into bf16 pairs and run
 * the encoder's tensor-core kernel (per (window, head), or persistent over head pairs when heads is even).
 * ALM_ERR_INVALID for null or host pointers, sizes < 1 or shift outside 0..6; ALM_ERR_UNSUPPORTED for C != 32 heads. */
ALM_API int alm_op_window_attention_ex(alm_ctx* ctx, const float* qkv, const float* bias_table, float* out_f32,
                                       void* out_hi, void* out_lo, int B, int nWh, int nWw, int C, int heads, int shift);
/* The same core on the operands the Swin blocks hand it: qkv as device bf16 planes qkv_hi / qkv_lo (uint16 buffers)
 * [B*nWh*nWw*49, 3C], the q columns already multiplied by 32^-0.5 (the encoder folds the scale into the qkv weight and
 * bias), so the kernel forms q k^T from the planes' values hi + lo with no further scaling.  Runs the encoder's
 * tensor-core kernel under the context's wattn_impl (3: persistent over head pairs when heads is even; 0 and 1: per
 * (window, head)); both read the lo plane at every nsplit.  bias_table, outputs and shift as in
 * alm_op_window_attention_ex.  qkv planes and out_f32 are aligned to 16 bytes, out_hi / out_lo to 8.  ALM_ERR_INVALID,
 * before any device work, for null (qkv_lo included) or host pointers, misalignment, sizes < 1 or shift outside 0..6;
 * ALM_ERR_UNSUPPORTED for C != 32 heads. */
ALM_API int alm_op_window_attention_planes(alm_ctx* ctx, const void* qkv_hi, const void* qkv_lo,
                                           const float* bias_table, float* out_f32, void* out_hi, void* out_lo, int B,
                                           int nWh, int nWw, int C, int heads, int shift);
/* The encoder's gather + LayerNorm + split (gather_ln).  Output row r (width C = nsrc * Cs) concatenates source rows
 * map[r * nsrc + s] (s = 0 .. nsrc - 1; -1 gives zeros; map NULL: row r * nsrc + s) of src f32 (row stride lds, the
 * first Cs values of each row are read).  gamma / beta [C] (NULL: no LayerNorm) normalise the row with eps.
 * zero_missing 1: a row whose sources are all -1 is written as +0 without LayerNorm or affine (the Swin pad tokens).
 * Outputs (each nullable, at least one): out_f32 (row stride ldo_f32) and the bf16 pair out_hi / out_lo (ldo_bf; out_lo
 * needs out_hi) of the row, and the second output y = row + add[r] (add f32 row stride ld_add, NULL: y = row) as the
 * pair out2_hi / out2_lo (ldo_bf) and / or out2_f32 (ldo_f32).  ld_add 0: one add row for every output row (the
 * decoder's query-position form).  Pointers are device memory (f32 16-byte aligned, bf16 8-byte); Cs and every row
 * stride a multiple of 4.  ALM_ERR_INVALID for other arguments, or a C that is neither a multiple of 128 nor 192;
 * ALM_ERR_UNSUPPORTED for a multiple of 128 the kernel has no instantiation for (only 128, 256, 384, 512, 768, 1024 and
 * 2048 are). */
ALM_API int alm_op_gather_ln(alm_ctx* ctx, const float* src, long lds, const int32_t* map, int nsrc, int Cs, long rows,
                             const float* gamma, const float* beta, float eps, int zero_missing, const float* add,
                             long ld_add, float* out_f32, long ldo_f32, void* out_hi, void* out_lo, long ldo_bf,
                             void* out2_hi, void* out2_lo, float* out2_f32);
/* alm_op_gather_ln as the joint polygon + recognition decoder pass runs it: rows 0 .. rows_half - 1 take gamma / beta /
 * add, rows rows_half .. rows - 1 take gamma2 / beta2 / add2 (each given exactly when its first-half twin is, same
 * layout).  ALM_ERR_INVALID unless nsrc == 1, Cs == 512 and 0 < rows_half < rows, and for what alm_op_gather_ln
 * rejects. */
ALM_API int alm_op_gather_ln_joint(alm_ctx* ctx, const float* src, long lds, const int32_t* map, int nsrc, int Cs,
                                   long rows, const float* gamma, const float* beta, float eps, int zero_missing,
                                   const float* add, long ld_add, float* out_f32, long ldo_f32, void* out_hi,
                                   void* out_lo, long ldo_bf, void* out2_hi, void* out2_lo, float* out2_f32,
                                   long rows_half, const float* gamma2, const float* beta2, const float* add2);
/* The encoder's int32 row maps over B images of an H x W token grid (rows numbered (b H + y) W + x), into map (device):
 *   kind 0, window: [B * nWh * nWw * 49], nWh = ceil(H / 7), nWw = ceil(W / 7); the token of (window, t) after zero pad
 *     to 7 nWh x 7 nWw, roll by -shift (0 .. 6) on both axes and 7 x 7 partition, or -1 for a pad token;
 *   kind 1, merge: [B * ceil(H / 2) * ceil(W / 2) * 4], the PatchMerging sources (2i, 2j), (2i + 1, 2j), (2i, 2j + 1),
 *     (2i + 1, 2j + 1) of output (i, j), or -1 past the grid;
 *   kind 2, nearest: [B * H * W], the source of F.interpolate(mode='nearest') from the ceil(H / 2) x ceil(W / 2) grid.
 * shift is 0 for kinds 1 and 2.  ALM_ERR_INVALID for other arguments. */
ALM_API int alm_op_swin_map(alm_ctx* ctx, int kind, int B, int H, int W, int shift, int32_t* map);
/* The 4 x 4 / stride-4 patch im2col of OmniParser's and MGP-STR's patch embedding.  img f32 [n_canvas, 3, Hc, Wc];
 * image b is the top-left H x W of canvas slot slots[b] (int32 device [B], each in 0 .. n_canvas - 1; NULL: slot b), and
 * nothing else of the canvas is read.  Out: the bf16 pair out_hi / out_lo (out_lo nullable) [B * ceil(H / 4) *
 * ceil(W / 4), 64] with k = c * 16 + ky * 4 + kx, zero past the image and in columns 48 .. 63.
 * ALM_ERR_INVALID for null or host pointers, H > Hc, W > Wc, sizes < 1 or a slot off the canvas. */
ALM_API int alm_op_patch_im2col(alm_ctx* ctx, const float* img, int n_canvas, int Hc, int Wc, const int32_t* slots, int B,
                                int H, int W, void* out_hi, void* out_lo);
/* The input_proj operand of an H x W page (fpn.py:38-44 and the stride-2 1 x 1 input_proj): p2 .. p5 f32 NHWC
 * [B, Hs[s], Ws[s], 256] on the stage grids of the page; out_hi / out_lo (out_lo nullable) [B * Hs[2] * Ws[2], 1024],
 * row (b, i, j) = [bilinear(p2), p3, bilinear(p4), bilinear(p5)] at (2i, 2j) of the p3 grid (align_corners = False).
 * ALM_ERR_INVALID for null or host pointers or sizes < 1. */
ALM_API int alm_op_fpn_assemble(alm_ctx* ctx, const float* p2, const float* p3, const float* p4, const float* p5, int B,
                                int H, int W, void* out_hi, void* out_lo);
/* Sine position embedding and key-padding mask at an h x w memory grid (position_embedding.py:24-44 on the mask
 * nearest-resized from H x W, swin_transformer.py:622): mask u8 [B, H, W] (1 = pad; NULL: no padding), pos f32
 * [B * h * w, 512] (y features, then x), kpm u8 [B * h * w].  dim_t is the model's own.  ALM_ERR_INVALID for null or host
 * pointers or sizes < 1; ALM_ERR_UNSUPPORTED when h * w > 25600 (the cumulative sums are held in shared memory). */
ALM_API int alm_op_sine_pos(alm_ctx* ctx, const uint8_t* mask, int B, int H, int W, int h, int w, float* pos,
                            uint8_t* kpm);
/* Row softmax over columns 0 .. n - 1 of s f32 (row stride lds), column j of row r excluded when
 * kpm[(r / rows_per_mask) * mask_ld + j] != 0 (kpm u8, NULL: no mask); out_f32 and / or the bf16 pair out_hi / out_lo
 * (out_lo needs out_hi), row stride ldo; columns n .. ldo - 1 are not written.  The kernel of MGP-STR's attention maps
 * and of the decoder's unfused cross-attention.  ALM_ERR_INVALID for null or host pointers, n < 1, lds or ldo < n,
 * or a mask with rows_per_mask < 1 or mask_ld < n. */
ALM_API int alm_op_softmax_rows(alm_ctx* ctx, const float* s, long lds, long rows, int n, const uint8_t* kpm,
                                int rows_per_mask, long mask_ld, float* out_f32, void* out_hi, void* out_lo, long ldo);
/* Decoder cross-attention of images img0 .. img0+nimg-1 (transformer.py:444-447, 8 heads of 64):
 * out[i, n] = softmax((q[i, n] / 8) K_i^T, keys with kpm != 0 excluded) V_i per head.
 * q f32 [nimg, Ncap, 512]; k, v f32 [nimg_total, M, 512] (already projected); kpm u8 [nimg_total, M] or NULL;
 * out f32 [nimg, Ncap, 512].  Builds the model's split-bf16 caches (K_c / V_c [img][96][M][64] with the data in the
 * 8 slices of decoder layer dl (0..11), and V^T [img][6144][Mpad] for xattn_impl 1), every element the call must not
 * read set to NaN, and runs the kernel the decoder runs for the context's xattn_impl / xattn_wg / xattn_ctas_per_sm /
 * nsplit, `launches` times on the same partial and counter buffers.  q_split 0: fp32 queries and output (the point
 * loop's form, Ncap <= 16); 1: split queries and output planes (the polygon / recognition form), re-joined into out.
 * ALM_ERR_UNSUPPORTED for xattn_impl 1 with Ncap > 1 (that path is the GEMM + softmax_rows pipeline). */
ALM_API int alm_op_cross_attention(alm_ctx* ctx, const float* q, const float* k, const float* v, const uint8_t* kpm,
                                   float* out, int nimg_total, int img0, int nimg, int Ncap, int M, int dl, int q_split,
                                   int launches);
/* alm_op_cross_attention with per-image live-key counts, the form pages of different sizes decode with: key_len host
 * [nimg_total], 1 <= key_len[i] <= M.  Keys at or beyond key_len[i] are NaN in the caches this call builds and must not
 * reach the output; the kernel's schedule covers ceil(key_len[i] / 64) key blocks of image i.
 * ALM_ERR_UNSUPPORTED for xattn_impl 1 (it masks with kpm only). */
ALM_API int alm_op_cross_attention_ex(alm_ctx* ctx, const float* q, const float* k, const float* v, const uint8_t* kpm,
                                      float* out, int nimg_total, int img0, int nimg, int Ncap, int M, int dl, int q_split,
                                      int launches, const int* key_len);
/* The character-location reduction of alm_omni_set_rec_locations on given operands: for every query row (image i,
 * query n) the centroid and central second moments (cx, cy, sxx, sxy, syy) of the head average of
 * softmax((q_h / 8) K_h^T) over the key positions (16 c + 8, 16 r + 8), (r, c) = (k / mw[i], k % mw[i]).
 * q f32 [nimg, Ncap, 512] (device); k f32 [nimg, M, 512] (device, already projected); kpm u8 [nimg, M] (device) or
 * NULL; key_len int host [nimg] (1 <= key_len[i] <= M) or NULL for M; mw int host [nimg] (>= 1); out f32
 * [nimg, Ncap, 5] (device).  Builds the split-bf16 K cache with the data in decoder layer 11's slices and NaN in every
 * element the kernel must not read (other layers, keys at or beyond key_len), and runs the decoder's kernel for the
 * context's nsplit.  q_split 0: fp32 queries (the one-query form); 1: split query planes (the Ncap > 1 form). */
ALM_API int alm_op_rec_locations(alm_ctx* ctx, const float* q, const float* k, const uint8_t* kpm, const int* key_len,
                                 const int* mw, float* out, int nimg, int Ncap, int M, int q_split);
/* The decoder's embedding at step t (transformer.py:313-328): x[s] = LayerNorm(word_emb[tokens[s * tstride + t]] +
 * pos_emb[t]) with gamma / beta (eps 1e-5), and qpos = pos_emb[t], the step's query position.  tokens int32, word_emb
 * f32 [V, 512], pos_emb f32 [1024, 512], x f32 [S, 512], qpos f32 [512].  S_half 0: the single form, tokens2 / pos_emb2
 * / qpos2 NULL.  0 < S_half < S: the joint polygon + recognition form, sequences S_half .. S - 1 are sequences
 * 0 .. S - S_half - 1 of tokens2 (row stride tstride2) with pos_emb2, and qpos2 = pos_emb2[t].  Device pointers (f32
 * 16-byte aligned).  ALM_ERR_INVALID for other arguments, t >= 1024, a row stride <= t, or a token outside [0, V). */
ALM_API int alm_op_embed_ln(alm_ctx* ctx, const int32_t* tokens, int tstride, int t, int S, int S_half,
                            const int32_t* tokens2, int tstride2, const float* word_emb, int V, const float* pos_emb,
                            const float* pos_emb2, const float* gamma, const float* beta, float* x, float* qpos,
                            float* qpos2);
/* One cached self-attention decode step at position t (transformer.py:439-441): qkv f32 [S, 1536] (q | k | v),
 * caches kc, vc f32 [S, Tmax, 512] (row t of both is written), out f32 [S, 512].  t < Tmax <= 1024; the kernel is
 * chosen from S and sattn_wide as in the decoder. */
ALM_API int alm_op_self_attention_step(alm_ctx* ctx, const float* qkv, float* kc, float* vc, float* out, int S, int t,
                                       int Tmax);
/* The same step as the beam-search loop runs it: key / value of position j < t of sequence s are read from cache row
 * anc[s * Tmax + j] (int32 [S, Tmax], device); row s supplies position t, which it writes. */
ALM_API int alm_op_self_attention_step_anc(alm_ctx* ctx, const float* qkv, float* kc, float* vc, float* out, int S, int t,
                                           int Tmax, const int32_t* anc);
/* Skinny fp32 linear of the decoder (M <= 32 rows): out[m, n] = act(xin[m] . W[n] + bias[n]) + resid[m, n], with
 * xin = x for columns n < n_split and x2 (NULL: x) for the rest.  x, x2 [M, K], W [N, K], resid and out [M, N].
 * ln_g / ln_b (K == 512): LayerNorm (eps 1e-5) of xin first, plus pos[K] for columns n < pos_split.
 * ALM_ERR_INVALID unless M <= 32, K % 4 == 0, K <= 512 or a multiple of 512 up to 2048, n_split % 4 == 0. */
ALM_API int alm_op_gemv(alm_ctx* ctx, const float* x, const float* x2, int n_split, const float* W, const float* bias,
                        const float* resid, float* out, int M, int N, int K, int act, const float* ln_g, const float* ln_b,
                        const float* pos, int pos_split);
/* Greedy token choice of one decode step (transformer.py:108-125,257-261,273-280): softmax over logits[s, :nsoft],
 * top-1 among the step's candidates (phase 0 = pt step gen_index, with a class slot when cfg->vie_categories > 0;
 * 1 = poly; 2 = rec), lowest id on ties.  logits f32 [S, V]; token int32 [S], prob f32 [S].  finished / ntok int32
 * [S] (both or neither) are updated as in the point loop: an EOS sets finished, another token sets
 * ntok = gen_index + 1, a finished sequence is left alone. */
ALM_API int alm_op_head_select(alm_ctx* ctx, const float* logits, int S, int V, int nsoft, int phase, int gen_index,
                               const alm_decode_cfg* cfg, int32_t* token, float* prob, int32_t* finished, int32_t* ntok);
/* One recognition beam step (the rule of alm_omni_set_rec_beams) over G groups of W rows: logits f32 [G*W, V].
 * score f32 [G*W] (in: parent scores, -inf = dead; out: child scores) and len int32 [G*W] (in / out: 0 = live, else the
 * length up to and including the terminal token) carry the state; gen_index 0 ignores them and starts from slot 0.
 * Out per child row: token int32, parent int32 (row of the parent within the group), prob f32 (0 for finished and
 * dead children; dead: token recog_pad, score -inf).  Device pointers. */
ALM_API int alm_op_beam_select(alm_ctx* ctx, const float* logits, int G, int W, int V, int nsoft, int gen_index,
                               const alm_decode_cfg* cfg, float* score, int32_t* len, int32_t* token, int32_t* parent,
                               float* prob);

/* ---- test-time image pipeline on the GPU (SURVEY 8f rank 1) ----------------------------------- */
/* Replaces RandomResize([test_min_size], test_max_size) -> ToTensor -> Normalize -> nested_tensor_from_tensor_list
 * (OCR/OmniParser/dataset/__init__.py:109-113, dataset/transforms.py:249-298,312-322, utils/nested_tensor.py:37-54)
 * for a batch of decoded 8-bit RGB pages.  The resize is Pillow's two-pass 8-bit bilinear resampling, reproduced bit
 * for bit (integer kernels; weights computed like Pillow computes them); ToTensor / Normalize are the same float32
 * operations, so tensors and mask equal the reference's.
 * alm_pre_omni_plan (host only): resized (h, w) per page = get_size_with_aspect_ratio, and the batch canvas.
 * alm_pre_omni_pages: rgb[i] = host or device pointer to page i, [heights[i]][widths[i]][3] uint8.  Outputs are
 * DEVICE buffers sized from the plan: tensors f32 [n,3,Hmax,Wmax] (zero padded), mask u8 [n,Hmax,Wmax] (1 = pad);
 * they feed alm_omni_encode directly. */
ALM_API int alm_pre_omni_plan(const int* heights, const int* widths, int n, int test_min_size, int test_max_size,
                              int* sizes /*[n][2] resized h, w*/, int* Hmax, int* Wmax);
/* Introspection (host only): the 22-bit fixed-point weights of ONE resampling pass exactly as the kernels use them
 * (filter 0 = bilinear, 1 = bicubic): bounds [out_size][2] = (first source index, taps), coefs [out_size][*ksize].
 * Call with coefs == NULL to obtain *ksize first (returns ALM_ERR_INVALID after storing it). */
ALM_API int alm_pre_coeffs(int in_size, int out_size, int filter, int* ksize, int* bounds, int* coefs, size_t cap_ints);
ALM_API int alm_pre_omni_pages(alm_ctx* ctx, const uint8_t* const* rgb, const int* heights, const int* widths, int n,
                               int test_min_size, int test_max_size, float* tensors, uint8_t* mask);
/* Replaces `img.resize((imgW, imgH), Image.BICUBIC)` + ToTensor (OCR/MGP-STR/demo.py:126-132, dataset.py:459-461):
 * out = DEVICE f32 [n,3,imgH,imgW] in [0,1], the input of alm_mgpstr_forward. */
ALM_API int alm_pre_mgp_crops(alm_ctx* ctx, const uint8_t* const* rgb, const int* heights, const int* widths, int n,
                              int imgH, int imgW, float* out);
/* Detected text regions -> recogniser inputs: replaces DocXChain's per-region loop of TextRecognition.order_point +
 * crop_image (Applications/DocXChain/modules/text_recognition.py:84-145: cv2.getPerspectiveTransform +
 * cv2.warpPerspective, INTER_LINEAR, BORDER_CONSTANT 0) followed by the resize + ToTensor of alm_pre_mgp_crops, bit for
 * bit, for R regions at once (three kernel launches whatever R is).
 * quads: HOST f32 [R][4][2] page pixel coordinates (x, y), any point order; page_index: HOST int32 [R] into the n_pages
 * pages rgb[i] (host or device, [heights[i]][widths[i]][3] uint8).  out: DEVICE f32 [R,3,imgH,imgW] in [0,1], the
 * input of alm_mgpstr_forward / alm_mgpstr_topk.  A crop whose truncated width or height is 0 is warped at its page's
 * size, as cv2 does for an empty dsize.  ALM_ERR_INVALID for a page index out of range, a non-finite coordinate,
 * imgH / imgW < 1, or crops that do not fit in the workspace (the message names the region).  R = 0 does nothing. */
ALM_API int alm_pre_quad_crops(alm_ctx* ctx, const uint8_t* const* rgb, const int* heights, const int* widths,
                               int n_pages, const float* quads, const int* page_index, int R, int imgH, int imgW,
                               float* out);
/* Introspection (host only): the per-region plan alm_pre_quad_crops uses.  ordered f32 [R][4][2] = order_point's
 * points, corners f32 [R][4][2] = crop_image's source corners, sizes int32 [R][2] = crop (width, height), minv f64
 * [R][9] = the inverse perspective map (crop pixel -> page).  Any output may be NULL. */
ALM_API int alm_pre_quad_plan(const int* heights, const int* widths, int n_pages, const float* quads,
                              const int* page_index, int R, float* ordered, float* corners, int* sizes, double* minv);
/* Curved text regions -> recogniser inputs: rectifies OmniParser's 16-point polygons (OCR/OmniParser/utils/misc.py:74-79:
 * 8 samples of the top boundary left -> right, then 8 of the bottom one right -> left) along the cubic Beziers of both
 * boundaries, then the resize + ToTensor of alm_pre_mgp_crops, for R regions at once (three kernel launches whatever
 * R is).  Per region:
 *   - each boundary's 8 points (as double) go through bezier_fit_quad (misc.py:81-110, a chord-length parametrised
 *     least-squares cubic; the pseudo-inverse drops eigenvalues <= 1e-15 x the largest, as np.linalg.pinv does).  A
 *     boundary whose segments sum to length 0 gets four control points equal to its first point;
 *   - crop width cw = int(mean of both boundaries' polyline lengths) + 1, height ch = int(mean of |p0 - p15| and
 *     |p7 - p8|) + 1;
 *   - column j at t = j / (cw - 1), row i at s = i / (ch - 1) (0 for a size of 1), T = top(t), B = bottom(1 - t),
 *     map = float32(T + (B - T) s), all in double with every operation rounded on its own;
 *   - the page is sampled as cv2.remap(page, map_x, map_y, INTER_LINEAR, BORDER_CONSTANT 0) does it, bit for bit.
 * polys: HOST f32 [R][16][2] page pixel coordinates (x, y); page_index: HOST int32 [R] into the n_pages pages rgb[i]
 * (host or device, [heights[i]][widths[i]][3] uint8).  out: DEVICE f32 [R,3,imgH,imgW] in [0,1], the input of
 * alm_mgpstr_forward / alm_mgpstr_topk.  ALM_ERR_INVALID for a page index out of range, a non-finite coordinate, a
 * control point with |value| >= 2^20, a crop side above 32766 (cv2.remap's limit), imgH / imgW < 1, or crops that do
 * not fit in the workspace (the message names the region).  R = 0 does nothing. */
ALM_API int alm_pre_curve_crops(alm_ctx* ctx, const uint8_t* const* rgb, const int* heights, const int* widths,
                                int n_pages, const float* polys, const int* page_index, int R, int imgH, int imgW,
                                float* out);
/* Introspection (host only): the per-region plan alm_pre_curve_crops uses.  ctrl f64 [R][2][4][2] = the control
 * points of the top and the bottom boundary, sizes int32 [R][2] = crop (width, height).  Any output may be NULL. */
ALM_API int alm_pre_curve_plan(const int* heights, const int* widths, int n_pages, const float* polys,
                               const int* page_index, int R, double* ctrl, int* sizes);
/* Window layout of text lines longer than MGP-STR's 4:1 input (host only).  sizes int32 [R][2]: each region's natural
 * crop (width cw, height ch) from alm_pre_quad_plan / alm_pre_curve_plan.  wn0 = ceil(ch 128 / 32) = 4 ch, overlap
 * ov = ch.  cw <= wn0: one window [0, cw), the plain crop.  Otherwise n = 1 + ceil((cw - wn0) / (wn0 - ov)) windows of
 * width wn = wn0; when that exceeds ALM_MAX_LINE_WINDOWS, n = 8 and wn = ceil((cw + 7 ov) / 8) (the windows are
 * compressed a little rather than the region refused).  Window i starts at x_i = min(i (wn - ov), cw - wn), so the
 * last one ends at cw and neighbours overlap by at least ch.  Outputs (any may be NULL): n int32 [R], x0 int32 [R][8]
 * (0 past n), wn int32 [R].  ALM_ERR_INVALID for a side < 1.  R = 0 does nothing. */
#define ALM_MAX_LINE_WINDOWS 8
ALM_API int alm_pre_line_windows(const int* sizes, int R, int* n, int* x0, int* wn);
/* Text lines -> recogniser inputs: the windows of alm_pre_line_windows of every region, in region order, for quads
 * (kind ALM_BOX_QUAD, regions f32 [R][4][2] as alm_pre_quad_crops) or 16-point polygons (ALM_BOX_CURVE, regions f32
 * [R][16][2] as alm_pre_curve_crops).  Window i of a region is columns [x_i, x_i + wn) of the crop alm_pre_quad_crops /
 * alm_pre_curve_crops cuts before resizing, bit for bit (the page-size fallback of a quad included), then Pillow's
 * bicubic resize of that wn x ch crop to 128 x 32 + ToTensor.  out: DEVICE f32 [sum of n][3][32][128].  Three kernel
 * launches whatever R is.  ALM_ERR_INVALID as alm_pre_quad_crops / alm_pre_curve_crops, and for an unknown kind.
 * R = 0 does nothing. */
ALM_API int alm_pre_line_crops(alm_ctx* ctx, const uint8_t* const* rgb, const int* heights, const int* widths,
                               int n_pages, int kind, const float* regions, const int* page_index, int R, float* out);
/* Turned recogniser inputs (DESIGN 4.13): region r of quads (kind ALM_BOX_QUAD, as alm_pre_quad_crops) or 16-point
 * polygons (ALM_BOX_CURVE, as alm_pre_curve_crops) read at turns[r] quarter-turns counter-clockwise.  lines 0: out
 * DEVICE f32 [R][3][32][128] = ToTensor(Image.fromarray(np.rot90(crop, q)).resize((128, 32), BICUBIC)), crop the
 * natural-size crop those entries cut (the page-size fallback of a quad included), bit for bit.  lines 1: the windows
 * of alm_pre_line_windows laid out on the turned crop's sides, cut from the turned crop as alm_pre_line_crops cuts
 * them, out [sum of windows][3][32][128].  Every turned pixel is the upright crop's pixel it came from; three kernel
 * launches whatever R and the turns.  ALM_ERR_INVALID for a turn outside 0..3, lines other than 0 / 1, and as
 * alm_pre_line_crops.  R = 0 does nothing. */
ALM_API int alm_pre_turned_crops(alm_ctx* ctx, const uint8_t* const* rgb, const int* heights, const int* widths,
                                 int n_pages, int kind, const float* regions, const int* page_index, int R,
                                 const int32_t* turns, int lines, float* out);
/* Tile layout of a page larger than OmniParser's input (host only; DESIGN 4.11).  tile T >= 64, overlap ov with
 * 0 <= 2 ov <= T.  Per axis of length L: L <= T gives one tile [0, L); otherwise n = 1 + ceil((L - T) / (T - ov)) tiles
 * at x_i = min(i (T - ov), L - T), so the last ends at L.  The page's tiles are the row-major product of both axes,
 * each min(T, H) x min(T, W).  Writes ny, nx; with y0 / x0 (either may be NULL) and cap >= max(ny, nx) also the
 * origins of the rows and the columns.  ALM_ERR_INVALID for a side < 1, a bad T / ov, or cap too small. */
ALM_API int alm_pre_omni_tile_plan(int H, int W, int tile, int overlap, int* ny, int* nx, int* y0, int* x0, int cap);
/* Tiles -> OmniParser inputs: tiles first .. first + count - 1 of the plan of every page (pages in order, each page's
 * tiles row-major), each cut from its page (one gather launch for all tiles) and put through alm_pre_omni_pages'
 * transform as an image of its own.  tensors / mask are the DEVICE outputs alm_pre_omni_pages gives for the sliced tiles
 * page[y0:y0+h, x0:x0+w], bit for bit (canvas: the largest resized tile).  ALM_ERR_INVALID for bad pages, T / ov or a
 * range outside the plan. */
ALM_API int alm_pre_omni_tiles(alm_ctx* ctx, const uint8_t* const* rgb, const int* heights, const int* widths,
                               int n_pages, int tile, int overlap, int first, int count, int test_min_size,
                               int test_max_size, float* tensors, uint8_t* mask);
/* Tiles by plan index: tiles index[0 .. count) of the plan (any order, repeats allowed), each as alm_pre_omni_tiles
 * cuts it, bit for bit; alm_pre_omni_tiles is this call with first .. first + count - 1.  ALM_ERR_INVALID for a null
 * index, count < 1, an index outside the plan and as alm_pre_omni_tiles. */
ALM_API int alm_pre_omni_tiles_at(alm_ctx* ctx, const uint8_t* const* rgb, const int* heights, const int* widths,
                                  int n_pages, int tile, int overlap, const int32_t* index, int count, int test_min_size,
                                  int test_max_size, float* tensors, uint8_t* mask);
/* Merge of the instances decoded from every tile of n_pages pages into page coordinates (DESIGN 4.11; the rule in full
 * is in tile_core.h).  Inputs, HOST buffers: the plan's tiles (n_tiles, pages in order, tiles row-major; tile_page
 * int32 [n_tiles] and tile_origin int32 [n_tiles][2] = (y0, x0) must be the plan's), and the decode of every tile in the
 * layout of alm_omni_decode: n_inst int32 [n_tiles], pt int64 [n_tiles][max_inst][2], poly [..][32], rec
 * [..][rec_length], rec_prob f32 [..][rec_length].  Per instance:
 *   - page coordinates of the point and the 16 vertices: origin + f32(f32(id / num_bins) * tile size), in double;
 *   - cut, and dropped, if a vertex lies within `margin` page pixels (<=) of an interior edge of its tile;
 *   - otherwise a candidate if its point lies in its tile's core, [s_{i-1}, s_i) per axis with the seams s_i =
 *     (x_{i+1} + x_i + T) / 2, widened by `band` on each interior side;
 *   - a candidate is dropped iff a candidate of a neighbouring tile of the same page (at most 8) has IoU of the
 *     vertices' bounding boxes >= iou (double) and ranks above it: larger distance d from its box to its own tile's
 *     interior edges (+inf without any), then lower tile index.
 * Outputs, HOST: page_count / page_offset int32 [n_pages], and the kept instances of every page in (tile, instance)
 * order at rows page_offset .. page_offset + page_count - 1: pts f64 [cap][2], polys f64 [cap][32], rec_out int64
 * [cap][rec_length], prob_out f32 [cap][rec_length], source int32 [cap][2] = (tile, instance).  cap >= sum(n_inst).
 * Three kernel launches whatever the counts.  ALM_ERR_INVALID, before any device work, for bad pages, T / ov, a margin
 * or band that is negative or not finite, iou outside (0, 1], a page index out of range, tiles that are not the plan's,
 * n_inst outside [0, max_inst], or cap too small. */
ALM_API int alm_omni_merge_tiles(alm_ctx* ctx, const int* heights, const int* widths, int n_pages, int tile,
                                 int overlap, int n_tiles, const int* tile_page, const int* tile_origin,
                                 const int32_t* n_inst, const int64_t* pt, const int64_t* poly, const int64_t* rec,
                                 const float* rec_prob, int max_inst, int rec_length, int num_bins, double margin,
                                 double band, double iou, int* page_count, int* page_offset, double* pts,
                                 double* polys, int64_t* rec_out, float* prob_out, int32_t* source, long cap);
/* Turned pages (DESIGN 4.14; the rule in full is in tile_core.h).  Page p of upright size H x W read at turns[p] = k
 * (0..3 counter-clockwise quarter-turns, np.rot90's convention) is read as np.rot90(page, k):
 *   - alm_pre_omni_tiles_turned: the plan is alm_pre_omni_tile_plan on the turned size (W x H for odd k), and every
 *     tile pixel is the page pixel np.rot90 takes it from.  tensors / mask are what alm_pre_omni_tiles gives for the
 *     host-turned pages, bit for bit.  One gather launch per call, then the resize passes.
 *   - alm_omni_merge_tiles_turned: heights / widths are the UPRIGHT sizes; tile_page / tile_origin are the turned
 *     pages' plan.  The merge runs in each turned page's frame exactly as alm_omni_merge_tiles (the kept rows and their
 *     order are those for np.rot90(page, k)), then the point and the 16 vertices of each kept row map to the page, in
 *     pixel-edge coordinates and one double operation per coordinate: k = 1: (W - v, u), k = 2: (W - u, H - v),
 *     k = 3: (v, H - u).  Vertex order is kept; rec / prob / source are unchanged.
 * ALM_ERR_INVALID, before any device work, for a null turns, a turn outside 0..3 and as the upright entries. */
ALM_API int alm_pre_omni_tiles_turned(alm_ctx* ctx, const uint8_t* const* rgb, const int* heights, const int* widths,
                                      int n_pages, const int32_t* turns, int tile, int overlap, int first, int count,
                                      int test_min_size, int test_max_size, float* tensors, uint8_t* mask);
ALM_API int alm_omni_merge_tiles_turned(alm_ctx* ctx, const int* heights, const int* widths, int n_pages,
                                        const int32_t* turns, int tile, int overlap, int n_tiles, const int* tile_page,
                                        const int* tile_origin, const int32_t* n_inst, const int64_t* pt,
                                        const int64_t* poly, const int64_t* rec, const float* rec_prob, int max_inst,
                                        int rec_length, int num_bins, double margin, double band, double iou,
                                        int* page_count, int* page_offset, double* pts, double* polys,
                                        int64_t* rec_out, float* prob_out, int32_t* source, long cap);
/* Turned tiles by plan index (DESIGN 4.21): tiles index[0 .. count) of the plan of the pages turned by turns[p]
 * (0..3; the plan alm_pre_omni_tiles_turned lays out, any order, repeats allowed), each cut as alm_pre_omni_tiles_turned
 * cuts it, bit for bit; alm_pre_omni_tiles_at is this call with every turn 0.  A page listed twice at two turns is two
 * pages of the plan.  ALM_ERR_INVALID for a null turns, a turn outside 0..3 and as alm_pre_omni_tiles_at. */
ALM_API int alm_pre_omni_tiles_at_turned(alm_ctx* ctx, const uint8_t* const* rgb, const int* heights, const int* widths,
                                         int n_pages, const int32_t* turns, int tile, int overlap, const int32_t* index,
                                         int count, int test_min_size, int test_max_size, float* tensors,
                                         uint8_t* mask);
/* Page orientation from four probe readings per page (DESIGN 4.14).  Inputs, HOST buffers: the decodes of 4 n_pages
 * readings in the layout of alm_omni_decode, reading 4 p + k = page p read whole at turn k: n_inst int32 [4 n_pages],
 * rec int64 [4 n_pages][max_inst][rec_length], rec_prob f32 [..].  An instance scores decode_pred_seq's 'score' (stop
 * at recog_pad_index or rec_eos_index, skip recog_pad_index - 1, sum(p) / (len + 1e-5) in double: what
 * alm_post_omni_spotting writes); a reading scores the sum of its instances' scores in instance order, in double (0
 * without instances).  Outputs, HOST: scores f64 [n_pages][4] and turns_out int32 [n_pages], the turn of the larger
 * score, the lower turn on a tie.  One kernel launch; only the turns and the scores are copied back.  ALM_ERR_INVALID,
 * before any device work, for n_pages / max_inst / rec_length < 1, a null buffer or n_inst outside [0, max_inst]. */
ALM_API int alm_omni_orient_select(alm_ctx* ctx, int n_pages, const int32_t* n_inst, const int64_t* rec,
                                   const float* rec_prob, int max_inst, int rec_length, int recog_pad_index,
                                   int rec_eos_index, int32_t* turns_out, double* scores);
/* Pages read at all four quarter-turns: the four readings of each page merged into one set of words (DESIGN 4.15; the
 * rule in full is in turn_core.h).  Inputs, HOST buffers, in the layout alm_omni_merge_tiles_turned writes for 4 n_pages
 * pages: reading r = 4 p + k is page p read at turn k, its rows are offset[r] .. offset[r] + count[r] - 1 (count /
 * offset int32 [4 n_pages], offset the exclusive prefix sum of count) of pts f64 [N][2], polys f64 [N][32], rec int64
 * [N][rec_length] and rec_prob f32 [N][rec_length], in page pixels.  Per row: box = the axis-aligned box of its 16
 * vertices (NaN when a vertex is not finite), s = decode_pred_seq's 'score' of its rec / rec_prob (as
 * alm_omni_orient_select), both in double.  A row is dropped iff a row of the same page at a different turn has box
 * IoU >= iou and ranks above it: larger s, then on equal s the lower turn.  Rows of one reading never suppress each
 * other.  Outputs, HOST: page_count / page_offset int32 [n_pages] and each page's kept rows in (turn, row) order,
 * copied unchanged, at rows page_offset .. page_offset + page_count - 1 of pts_out f64 [cap][2], polys_out [cap][32],
 * rec_out int64 [cap][rec_length], prob_out f32 [cap][rec_length], with source int32 [cap][2] = (turn, index within
 * that reading).  Three kernel launches whatever the counts; only the kept rows and the per-page counts are copied
 * back.  ALM_ERR_INVALID, before any device work, for n_pages or rec_length < 1, a null buffer, a negative count,
 * offsets that are not the exclusive prefix sum of the counts, iou outside (0, 1] or not finite, or cap below the
 * sum of the counts. */
ALM_API int alm_omni_merge_turns(alm_ctx* ctx, int n_pages, const int32_t* count, const int32_t* offset,
                                 const double* pts, const double* polys, const int64_t* rec, const float* rec_prob,
                                 int rec_length, int recog_pad_index, int rec_eos_index, double iou,
                                 int32_t* page_count, int32_t* page_offset, double* pts_out, double* polys_out,
                                 int64_t* rec_out, float* prob_out, int32_t* source, long cap);
/* The same merge over n_readings readings per page (1 <= n_readings <= 64): reading r = n_readings p + k is page p's
 * reading k, "turn" above reads "reading index k", and source = (k, index within that reading).  alm_omni_merge_turns
 * is n_readings = 4, with the same outputs and launches.  The window readings of a dense page (alm_omni_decode_dense,
 * DESIGN 4.16) are merged with this rule, reading k = window k, boxes in coordinate bins.  Errors as
 * alm_omni_merge_turns, and ALM_ERR_INVALID for n_readings outside 1..64. */
ALM_API int alm_omni_merge_readings(alm_ctx* ctx, int n_pages, int n_readings, const int32_t* count,
                                    const int32_t* offset, const double* pts, const double* polys, const int64_t* rec,
                                    const float* rec_prob, int rec_length, int recog_pad_index, int rec_eos_index,
                                    double iou, int32_t* page_count, int32_t* page_offset, double* pts_out,
                                    double* polys_out, int64_t* rec_out, float* prob_out, int32_t* source, long cap);
/* Words that cross tile seams, recovered from a whole-page reading of each page (DESIGN 4.17; the rule in full is in
 * whole_core.h).  A word wider than the overlap that crosses a seam is cut in every tile it touches, so the tile merge
 * drops it; a reading of the whole page sees it whole.  Page p of upright size heights[p] x widths[p], read at
 * turns[p] (null = all upright), tiled with (tile, overlap) and merged by alm_omni_merge_tiles(_turned).  Inputs, HOST
 * buffers:
 *   - tile rows: what alm_omni_merge_tiles(_turned) wrote for the pages: count / offset int32 [n_pages] (offset the
 *     exclusive prefix sum of count), pts f64 [N][2], polys f64 [N][32], rec int64 [N][rec_length], rec_prob f32
 *     [N][rec_length], source_in int32 [N][2], in page pixels;
 *   - whole rows: each page's whole-page reading (np.rot90(page, turn) decoded as one image) in the layout of
 *     alm_omni_decode / alm_omni_decode_dense with cap_in slots per page: n_inst int32 [n_pages] in [0, cap_in], pt
 *     int64 [n_pages][cap_in][2], poly [..][32], whole_rec [..][rec_length], whole_prob f32 [..][rec_length];
 *     coordinates f32(f32(id / num_bins) * turned size), origin 0, in the turned frame.
 * A whole row is kept iff every tile of the page's plan cuts it: a vertex within margin (<=) of an interior edge of that
 * tile, in its frame, vertices outside the tile included (alm_omni_merge_tiles' cut).  Its point and vertices then map
 * back to the page as alm_omni_merge_tiles_turned maps them.  A tile row is dropped iff its point lies inside the
 * 16-vertex polygon of a kept whole row of its page (crossing-number rule in double; a NaN coordinate is never inside).
 * Whole rows never drop each other.  Outputs, HOST: page_count / page_offset int32 [n_pages] and each page's kept tile
 * rows in input order, then its kept whole rows in instance order, at rows page_offset .. page_offset + page_count - 1
 * of pts_out f64 [cap][2], polys_out [cap][32], rec_out int64 [cap][rec_length], prob_out f32 [cap][rec_length], with
 * source int32 [cap][2] = source_in's (tile, instance) for tile rows and (-1, instance) for whole rows.  A page that fits
 * in one tile keeps its tile rows and no whole row.  Three kernel launches whatever the counts; only the kept rows and
 * the per-page counts are copied back.  ALM_ERR_INVALID, before any device work, for bad pages, tile / overlap, a margin
 * that is negative or not finite, a turn outside 0..3, num_bins / rec_length / cap_in < 1, a null buffer, a negative
 * count, offsets that are not the exclusive prefix sum of the counts, n_inst outside [0, cap_in], or cap below sum(count)
 * + sum(n_inst). */
ALM_API int alm_omni_merge_whole_page(alm_ctx* ctx, const int* heights, const int* widths, int n_pages,
                                      const int32_t* turns, int tile, int overlap, double margin, int num_bins,
                                      const int32_t* count, const int32_t* offset, const double* pts,
                                      const double* polys, const int64_t* rec, const float* rec_prob,
                                      const int32_t* source_in, const int32_t* n_inst, const int64_t* pt,
                                      const int64_t* poly, const int64_t* whole_rec, const float* whole_prob,
                                      int cap_in, int rec_length, int32_t* page_count, int32_t* page_offset,
                                      double* pts_out, double* polys_out, int64_t* rec_out, float* prob_out,
                                      int32_t* source, long cap);
/* One box per recognised character of words read in tiles, turned or not, in page pixels (DESIGN 4.20; the rule in
 * full is in rec_box_core.h): the counterpart of postprocess.rec_char_boxes for spot_tiled and read_regions.  Inputs,
 * HOST buffers, word n of n_words: polys f64 [n_words][32] (its 16 vertices in page pixels, as the merges return
 * them), rec int64 [n_words][rec_length], loc f32 [n_words][rec_length][5] (the character locations of the tile
 * instance it came from, (cx, cy, sxx, sxy, syy) normalised by that image's encoded size) and frame_index int32
 * [n_words] into frames int32 [n_frames][7] = (H, W, turn, y0, x0, h, w): the upright page size, the turn the page was
 * read at and the tile's origin and size in the turned page (a page read whole: 0, 0 and the page's size, turn 0).
 *   centre  (x0 + cx w, y0 + cy h) in double, mapped to the upright page as alm_omni_merge_tiles_turned maps points;
 *   cov     (sxx w w, sxy w h, syy h h), turned with the page: an odd turn swaps sxx and syy and negates sxy;
 *   chars   the steps decode_seq keeps: stop at recog_pad_index or rec_eos_index, skip recog_pad_index - 1;
 *   box     rec_char_boxes' rule on the page polygon: nearest point q of the centre line (P_i + P_{15-i}) / 2, unit
 *           direction u of that segment, local height H, half-width a = sqrt(3) sqrt(u^T cov u); corners q -+ a u -+
 *           (H / 2) v, v = (-u_y, u_x), top-left, top-right, bottom-right, bottom-left in reading direction.
 * Every operation in double, rounded on its own; non-finite inputs propagate as NaN.  Outputs, HOST: n_chars int32
 * [n_words]; per slot [n_words][rec_length] (character i of word n is slot i) step int32 (the rec step it came
 * from), centre f64 [2], cov f64 [3] = (sxx, sxy, syy) and box f64 [8] = four corners (x, y); slots past n_chars are
 * 0.  One kernel launch whatever n_words is (one warp per word, no atomics: bit-reproducible), none for n_words = 0.
 * ALM_ERR_INVALID, before any device work, for n_words < 0, rec_length outside 1..1021, a null buffer or n_frames < 1
 * (with n_words > 0), a frame index out of range, a turn outside 0..3, a non-positive size or a tile outside its
 * turned page. */
ALM_API int alm_omni_char_boxes(alm_ctx* ctx, long n_words, int rec_length, const double* polys, const int64_t* rec,
                                const float* loc, const int32_t* frame_index, int n_frames, const int32_t* frames,
                                int recog_pad_index, int rec_eos_index, int32_t* n_chars, int32_t* step,
                                double* centre, double* cov, double* box);
/* Caller-given regions read at quarter-turns: of each region's candidate readings the one kept, and its point and
 * polygon in upright page pixels (DESIGN 4.21; the rule in full is in region_turn_core.h).  Inputs, HOST buffers:
 * n_regions regions of n_cand (1..4) candidate readings each, candidate c of region r read by alm_omni_decode_at in
 * the frame frames[frame_index[r][c]], frames int32 [n_frames][7] = (H, W, turn, y0, x0, h, w) as alm_omni_char_boxes
 * takes them (one frames array serves both calls); pt int64 [n_regions][n_cand][2] and poly [..][32] in bins of that
 * frame, rec [..][rec_length] and rec_prob f32 [..][rec_length].
 *   score  decode_pred_seq's 'score' of each candidate's rec / rec_prob (as alm_omni_orient_select scores an instance);
 *   keep   the candidate of the largest score, on equal scores the lower turn, then the lower index; a NaN score never
 *          ranks above another and every other ranks above it;
 *   map    the kept candidate's point and 16 vertices: y0 / x0 + f32(f32(id / num_bins) * h / w) in double, as
 *          alm_omni_merge_tiles maps a tile's reading, then to the upright page as alm_omni_merge_tiles_turned maps a
 *          turned row, vertex order kept.  Turn 0 with one candidate is the tile merge's mapping alone.
 * Outputs, HOST: kept int32 [n_regions] (the candidate index), scores f64 [n_regions][n_cand], pts f64 [n_regions][2]
 * and polys f64 [n_regions][32].  One kernel launch whatever n_regions is (one warp per region, no atomics:
 * bit-reproducible), none for n_regions = 0.  ALM_ERR_INVALID, before any device work, for n_regions < 0, n_cand
 * outside 1..4, rec_length outside 1..1021, num_bins < 1, a null buffer or n_frames < 1 (with n_regions > 0), a frame
 * index out of range, a turn outside 0..3, a non-positive size or a tile outside its turned page. */
ALM_API int alm_omni_select_regions(alm_ctx* ctx, long n_regions, int n_cand, const int32_t* frame_index, int n_frames,
                                    const int32_t* frames, const int64_t* pt, const int64_t* poly, const int64_t* rec,
                                    const float* rec_prob, int rec_length, int num_bins, int recog_pad_index,
                                    int rec_eos_index, int32_t* kept, double* scores, double* pts, double* polys);
/* KIE on pages larger than the model's input or turned by quarter-turns: the entities decoded from every tile merged
 * into page coordinates on the device (DESIGN 4.18; the rule in full is in kie_tile_core.h).  Page p of upright size
 * heights[p] x widths[p], read as np.rot90(page, turns[p]) (turns null = all upright), tiled with (tile, overlap) as
 * alm_pre_omni_tile_plan lays the turned page out.  Inputs, HOST buffers, one row per tile of the plan (tile_page /
 * tile_origin as alm_omni_merge_tiles takes them), in the layout of alm_omni_decode_kie: n_tok int32 [n_tiles] in
 * [0, max_tok], tokens int64 [n_tiles][max_tok], tok_prob f32 [..], n_inst int32 [n_tiles] in [0, max_inst], inst_pos
 * int32 [n_tiles][max_inst], poly int64 [n_tiles][max_inst][32].  Each tile was read as an image of its own, with
 * orig_size = the tile's (h, w).
 *   1. Entities of a tile: the walk of decode_vie_pt_poly_rec_seq (transformer.py:148-215): an (x, y) pair of bins is
 *      a word, a lone bin is skipped, any other token closes an entity with class token - class_base and probability
 *      tok_prob[i].  An entity's words are a run of consecutive instances; words after the last class token belong to
 *      no entity and are dropped.
 *   2. Geometry, in double, one rounding per operation: word rect in page pixels x0 + (w min_x_id) / num_bins (the
 *      product an exact integer), the same for y and the maxima; entity box the union of its words' rects; anchor the
 *      centre of the box.  cut: the box within margin (<=) of an interior edge of its tile.  cand: not cut, and the
 *      anchor in the tile's core widened by band (alm_omni_merge_tiles' core).  d: the distance from the box to the
 *      tile's nearest interior edge (+inf without one).
 *   3. Keep: a candidate entity is dropped iff a candidate entity of a neighbouring tile of the same page has box IoU
 *      >= iou and ranks above it (larger d, then lower tile index): alm_omni_merge_tiles' rule at entity granularity.
 *      The class plays no part; entities of one tile never suppress each other.
 *   4. An entity without words has no box: kept on a page that is one tile, dropped on a page of several tiles.
 *   5. Turned pages: the merge runs in the turned frame; each kept word rect maps back corner by corner as
 *      alm_omni_merge_tiles_turned maps points, min / max re-ordered; each polygon vertex by vertex, order kept.
 * On a page that is one upright tile the result is alm_post_omni_kie_json's entity list, rects bit for bit.
 * Outputs, HOST: page_count / page_offset int32 [n_pages]: page p's kept entities are rows page_offset[p] .. +
 * page_count[p] - 1, in (tile, entity) order, of ent_class int32 [cap_ent] (class index, token - class_base), ent_prob
 * f32, word_offset / word_count int32 (the entity's words are word rows word_offset .. + word_count - 1, in decode
 * order) and ent_source int32 [cap_ent][2] = (tile, entity index in that tile); word_rect f64 [cap_words][4] (x0, y0,
 * x1, y1), word_poly f64 [cap_words][32] (the 16 vertices, decode_pred_seq's coordinates plus the tile origin, mapped
 * back) and word_source int32 [cap_words][2] = (tile, instance), in page pixels of the upright page.  Four kernel
 * launches whatever the counts; only the kept rows and the per-page counts are copied back.  ALM_ERR_INVALID, before
 * any device work, for everything alm_omni_merge_tiles refuses, a turn outside 0..3, max_tok / max_inst / num_bins /
 * n_classes < 1, n_tok outside [0, max_tok], an inst_pos that does not list the (x, y) pairs of the token stream, a
 * token that is neither a bin nor a class in [0, n_classes), or cap_ent / cap_words below all entities / all their
 * words. */
ALM_API int alm_omni_merge_kie_tiles(alm_ctx* ctx, const int* heights, const int* widths, int n_pages,
                                     const int32_t* turns, int tile, int overlap, int n_tiles, const int* tile_page,
                                     const int* tile_origin, const int32_t* n_tok, const int64_t* tokens,
                                     const float* tok_prob, int max_tok, const int32_t* n_inst,
                                     const int32_t* inst_pos, const int64_t* poly, int max_inst, int num_bins,
                                     int class_base, int n_classes, double margin, double band, double iou,
                                     int32_t* page_count, int32_t* page_offset, int32_t* ent_class, float* ent_prob,
                                     int32_t* word_offset, int32_t* word_count, int32_t* ent_source, long cap_ent,
                                     double* word_rect, double* word_poly, int32_t* word_source, long cap_words);
/* KIE entities that cross tile seams, recovered from a whole-page KIE reading of each page (DESIGN 4.22; the rule in
 * full is in kie_whole_core.h).  An entity taller or wider than the overlap that crosses a seam is cut in every tile,
 * so alm_omni_merge_kie_tiles drops it; a reading of the whole page sees it whole.  Page p of upright size heights[p] x
 * widths[p], read at turns[p] (null = all upright), tiled with (tile, overlap) and merged by alm_omni_merge_kie_tiles.
 * Inputs, HOST buffers:
 *   - tile entities: what alm_omni_merge_kie_tiles wrote for the pages: count / offset int32 [n_pages] (offset the
 *     exclusive prefix sum of count), ent_class int32 [E], ent_prob f32 [E], word_offset / word_count int32 [E]
 *     (word_offset the exclusive prefix sum of word_count), ent_source int32 [E][2]; word_rect f64 [N][4], word_poly
 *     f64 [N][32], word_source int32 [N][2], in page pixels;
 *   - whole readings: each page's whole-page KIE reading (np.rot90(page, turn) decoded as one image, orig_size its
 *     turned size) in the layout of alm_omni_decode_kie, one row per page: n_tok int32 [n_pages] in [0, max_tok],
 *     tokens int64 [n_pages][max_tok], tok_prob f32 [..], n_inst int32 [n_pages] in [0, max_inst], inst_pos int32
 *     [n_pages][max_inst], poly int64 [n_pages][max_inst][32].
 * Whole entities: alm_omni_merge_kie_tiles' walk (1.) and word rects (2.) with the turned page's size and origin 0, box
 * the union of the word rects.  A whole entity is kept iff it has words and every tile of the page's plan cuts its box:
 * an edge within margin (<=) of an interior edge of that tile, in its frame, edges outside the tile included.  Its word
 * rects then map back to the page corner by corner, min / max re-ordered, its polygons vertex by vertex, as
 * alm_omni_merge_kie_tiles maps turned words.  A tile entity is dropped iff its anchor (the centre of the union of its
 * word rects) lies inside the box of a kept whole entity of its page, edges included, in double, in page pixels; a NaN
 * or non-finite coordinate is never inside, and an entity without words is never dropped.  Whole entities never drop
 * each other.  Outputs, HOST, in alm_omni_merge_kie_tiles' layout: page p's kept tile entities in input order, then its
 * kept whole entities in entity order; ent_source_out = ent_source's (tile, entity) for tile entities and (-1, entity)
 * for whole ones, word_source_out = (tile, instance) and (-1, instance).  A page that fits in one tile keeps its tile
 * entities and no whole entity.  Three kernel launches whatever the counts; only the kept rows and the per-page counts
 * are copied back.  ALM_ERR_INVALID, before any device work, for bad pages, tile / overlap, a margin that is negative
 * or not finite, a turn outside 0..3, max_tok / max_inst / num_bins / n_classes < 1, a null buffer, a negative count,
 * offsets that are not the exclusive prefix sums of their counts, a whole reading alm_omni_merge_kie_tiles would refuse
 * as a tile's (n_tok, n_inst, inst_pos, tokens), or cap_ent / cap_words below the tile entities plus the whole
 * entities / all their words. */
ALM_API int alm_omni_merge_kie_whole_page(
    alm_ctx* ctx, const int* heights, const int* widths, int n_pages, const int32_t* turns, int tile, int overlap,
    double margin, int num_bins, int class_base, int n_classes, const int32_t* count, const int32_t* offset,
    const int32_t* ent_class, const float* ent_prob, const int32_t* word_offset, const int32_t* word_count,
    const int32_t* ent_source, const double* word_rect, const double* word_poly, const int32_t* word_source,
    const int32_t* n_tok, const int64_t* tokens, const float* tok_prob, int max_tok, const int32_t* n_inst,
    const int32_t* inst_pos, const int64_t* poly, int max_inst, int32_t* page_count, int32_t* page_offset,
    int32_t* ent_class_out, float* ent_prob_out, int32_t* word_offset_out, int32_t* word_count_out,
    int32_t* ent_source_out, long cap_ent, double* word_rect_out, double* word_poly_out, int32_t* word_source_out,
    long cap_words);
/* Spotted words -> text lines in reading order, each with a 16-point line polygon (DESIGN 4.12; the rule in full is
 * in group_core.h).  Inputs, HOST buffers, in the layout alm_omni_merge_tiles writes: page p's words are rows
 * page_offset[p] .. page_offset[p] + page_count[p] - 1 of polys f64 [N][32], N = the sum of page_count; the rows of
 * all pages partition [0, N).  A word is 16 vertices (x, y) in page pixels, top boundary P0 -> P7 left to right, bottom
 * P8 -> P15 right to left.  All arithmetic in double, every operation rounded on its own.  Per word:
 *   - frame: left end L = (P0 + P15) / 2, right end R = (P7 + P8) / 2, direction u = (R - L) / |R - L|, normal
 *     n = (-u.y, u.x), height h = (|P0 - P15| + |P7 - P8|) / 2.  A word with a non-finite vertex, or whose |R - L| or
 *     h is zero or not finite, is degenerate: a line of its own.
 *   - j is a successor candidate of i (same page, neither degenerate) when, with d = L_j - R_i, gap = d . u_i,
 *     off = d . n_i, hmin / hmax = min / max(h_i, h_j): -max_overlap hmin <= gap <= max_gap hmax, |off| <= max_offset
 *     hmin, hmin >= height_ratio hmax and u_i . u_j >= cos_tol.
 *   - succ(i) = the candidate with the smallest (max(gap, 0), |off|, j); pred(j) = of the i that have j as a
 *     candidate, the smallest (max(gap, 0), |off|, i).  i -> j is a link iff succ(i) = j and pred(j) = i.  Links form
 *     chains, and cycles for text on a closed curve; a cycle is opened by dropping the link into its lowest row.
 * A line is a chain, its words ranked from its head.  The lines of a page are ordered by (L.y, L.x, row) of their
 * head (L = (+inf, +inf) for a word with a non-finite vertex), pages in order.  The line polygon, in the words' own
 * format: the words' top boundaries concatenated in order, and their bottom boundaries taken left to right, each
 * resampled at 8 points of equal arc length (the first and the last point kept; a polyline of length 0 repeats its
 * first point), top left -> right then bottom right -> left; the line of a degenerate word gets that word's polygon.
 * Outputs, HOST: n_lines / line_offset int32 [n_pages] (page p's lines are line_offset[p] .. + n_lines[p] - 1);
 * per line l its words are order[line_first[l] .. line_first[l] + line_words[l] - 1] (word rows; page p's part of
 * order occupies the page's own row range) and line_polys f64 [cap][32] its polygon; per word row line_of (its line)
 * and rank_of (its place in the line).  cap >= N.  Five kernel launches whatever the counts (none when N = 0: empty
 * pages have zero lines).  ALM_ERR_INVALID, before any device work, for n_pages < 1, a null buffer, a negative count,
 * rows that overlap or leave [0, N), cos_tol outside [-1, 1], height_ratio outside [0, 1], max_offset / max_overlap /
 * max_gap negative or not finite, or cap < N; the message names the argument.  Proposed parameters: cos 15 degrees,
 * 0.5, 0.5, 0.5, 1.5. */
ALM_API int alm_omni_group_lines(alm_ctx* ctx, int n_pages, const int* page_count, const int* page_offset,
                                 const double* polys, double cos_tol, double height_ratio, double max_offset,
                                 double max_overlap, double max_gap, int* n_lines, int* line_offset, int* line_first,
                                 int* line_words, int32_t* order, int32_t* line_of, int32_t* rank_of,
                                 double* line_polys, long cap);

/* ---- post-processing (host only: no context, no GPU; SURVEY 8f rank 2) ------------------------ */
/* Sequences -> structured result, the step right after the forward.  Errors: negative ALM_ERR_*; the message of
 * the last failing call of the calling thread is returned by alm_post_last_error(). */
ALM_API const char* alm_post_last_error(void);

/* Replaces decode_pred_seq + decode_seq (OCR/OmniParser/engine/val.py:70-100, utils/misc.py:147-189) for ONE image:
 *   pt [2*n] / poly [32*n] / rec [n*rec_length] int64 ids and rec_prob [n*rec_length] f32 as returned by
 *   alm_omni_decode (one row of its outputs); chars = args.chars as UTF-8 (one code point per class id
 *   num_bins + i); orig_h / orig_w = target['orig_size'].
 * Outputs (caller buffers): pts [n,2] and polys [n,32] doubles holding the reference's float32 values
 * (id / num_bins * size, both steps rounded to f32 like the torch expressions), scores [n] doubles
 * (sum(p) / (len + 1e-5) in double), texts: n NUL-terminated UTF-8 strings at stride text_stride bytes. */
ALM_API int alm_post_omni_spotting(const int64_t* pt, const int64_t* poly, const int64_t* rec, const float* rec_prob, int n,
                                   int rec_length, int num_bins, int recog_pad_index, int rec_eos_index, const char* chars,
                                   long orig_h, long orig_w, double* pts, double* polys, double* scores, char* texts,
                                   size_t text_stride);
/* The same results as the JSON text `json.dumps(results, indent=4)` writes for this image (val.py:63-67; keys
 * image_id, pts, score, polys, rec; Python float repr; ensure_ascii escapes).  Writes at most cap bytes incl. NUL
 * and always stores the needed size (incl. NUL) in *needed; returns ALM_ERR_INVALID if cap is too small. */
ALM_API int alm_post_omni_json(const int64_t* pt, const int64_t* poly, const int64_t* rec, const float* rec_prob, int n,
                               int rec_length, int num_bins, int recog_pad_index, int rec_eos_index, const char* chars,
                               long orig_h, long orig_w, const char* image_id, char* json, size_t cap, size_t* needed);

/* KIE: the entity walk of decode_vie_pt_poly_rec_seq (OCR/OmniParser/model/transformer.py:148-215) over ONE image's
 * outputs of alm_omni_decode_kie (tokens / probs [n_tok], inst_pos [n_inst], poly [n_inst,32], rec [n_inst,rec_length]),
 * written as the JSON text `json.dump(output, f)` stores (engine/val.py:38-42):
 * [[text, class_name, prob, [[x0, y0, x1, y1], ...]], ...].  classes[i] names token id class_base + i
 * (class_base = padding_index + 1, transformer.py:54-61).  Size protocol as alm_post_omni_json. */
ALM_API int alm_post_omni_kie_json(const int64_t* tokens, const float* probs, int n_tok, const int32_t* inst_pos, int n_inst,
                                   const int64_t* poly, const int64_t* rec, int rec_length, int num_bins,
                                   int recog_pad_index, int rec_eos_index, const char* chars, const char* const* classes,
                                   int n_classes, int class_base, long orig_h, long orig_w, char* json, size_t cap,
                                   size_t* needed);

/* MGP-STR A^3 fusion (OCR/MGP-STR/test_final.py:176-240, demo.py:36-112, utils.py:52-87) for B crops.
 *   ids / prob: [3][B,T] int32 top-1 ids and f32 max-softmax probabilities of the char, bpe and wp heads INCLUDING
 *   position 0 (exactly what alm_mgpstr_forward returns; T = 27).
 *   tables: token strings per id, UTF-8 -- char: ['[GO]', '[s]'] + opt.character; bpe: the byte-decoded GPT-2 token
 *   strings; wp: the WordPiece tokens of bert-base-uncased.  (The reference obtains them from the HuggingFace
 *   tokenizers; they are data, passed in by the caller.)
 * Per crop and head: text (pruned at the end-of-sentence marker the way the reference prunes it -- string find of
 * '[s]' / '#' / '[SEP]', including its -1 quirk) and confidence = cumprod of the max-probs up to the EOS position
 * (first id 1 / 2 / 102 for char / bpe / wp; char uses the STRING index like the reference); fused = the head with
 * the largest confidence (strictly greater, in char, bpe, wp order; none if all are 0).
 * Outputs: texts [3][B] and fused [B] strings at stride text_stride; conf [3][B] f32; source [B] int32 (0 char, 1 bpe,
 * 2 wp, -1 none). */
ALM_API int alm_post_mgp_fuse(const int32_t* ids, const float* prob, int B, int T, const char* const* char_table, int n_char,
                              const char* const* bpe_table, int n_bpe, const char* const* wp_table, int n_wp, char* texts,
                              char* fused, size_t text_stride, float* conf, int32_t* source);

#ifdef __cplusplus
}
#endif
#endif /* ALM_OCR_H_ */
