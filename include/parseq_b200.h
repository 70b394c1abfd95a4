/*
 * parseq_b200.h - C ABI of the H100-native (sm_90a) PARSeq inference engine (libparseq_b200.so).
 *
 * The reference (baudm/parseq) has no FFI / plugin boundary for this path: it sits behind the Python
 * class strhub.models.parseq.system.PARSeq (system.py:33-88) wrapping the nn.Module
 * strhub.models.parseq.model.PARSeq (model.py:31-169).  Each entry point below states the reference
 * method it replaces.  All pointers are plain device or host pointers; no torch types cross this
 * boundary.  All functions return 0 on success and a negative parseq_status on failure;
 * parseq_last_error() returns a human-readable message for the calling thread's last failure.
 *
 * Threading / streams: an engine handle is NOT thread-safe (one handle per device and stream user).
 * All work is enqueued on the caller's stream; the only host synchronisation is inside
 * parseq_forward_host (which must return host-visible results), parseq_finalize and a
 * parseq_forward_crops_oriented call with a min_confidence.
 */
#ifndef PARSEQ_B200_H_
#define PARSEQ_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct parseq_engine parseq_engine;
typedef void* parseq_stream_t;           /* cudaStream_t */

typedef enum parseq_status {
  PARSEQ_OK = 0,
  PARSEQ_ERR_INVALID_ARG = -1,
  PARSEQ_ERR_UNSUPPORTED = -2,           /* configuration outside what the kernels cover */
  PARSEQ_ERR_CUDA = -3,
  PARSEQ_ERR_STATE = -4,                 /* e.g. forward before finalize, missing weight */
  PARSEQ_ERR_NO_DEVICE = -5              /* no sm_90 device: there is NO CPU fallback */
} parseq_status;

/* Architecture hyper-parameters: the ctor arguments of model.PARSeq (model.py:33-49) /
 * system.PARSeq (system.py:35-60).  num_tokens = len(tokenizer) = charset + EOS + BOS + PAD. */
typedef struct parseq_config {
  int32_t img_h, img_w;                  /* img_size     */
  int32_t patch_h, patch_w;              /* patch_size   */
  int32_t embed_dim;
  int32_t enc_num_heads, enc_mlp_ratio, enc_depth;
  int32_t dec_num_heads, dec_mlp_ratio, dec_depth;   /* dec_depth >= 1 decoder layers (1 in every reference config) */
  int32_t max_label_length;              /* 25 -> 26 decode positions; 0..63 (labels of up to 63 characters) */
  int32_t num_tokens;                    /* 97: EOS=0, chars 1..94, BOS=95, PAD=96 (data/utils.py:102-111); 4..16386
                                            (at most 16384 head classes, e.g. CJK charsets) */
  int32_t max_batch;                     /* images per super-chunk / CUDA graph (workspace sizing); 0 = 512 */
  int32_t device;                        /* CUDA device ordinal */
  int32_t arch;                          /* 0: PARSeq (parseq/model.py); 1: ViTSTR (vitstr/model.py:14-28: the same ViT with
                                          * a class token and a per-token head; the dec_* fields are ignored) */
} parseq_config;

/* Replaces model.PARSeq.__init__ (model.py:33-71): allocates device weights + workspace.
 * arch = 1 replaces vitstr/system.py:50-59 (ViTSTR(VisionTransformer) ctor): state_dict keys are then those of the
 * timm ViT itself ("cls_token", "pos_embed" [1, T+1, D], "patch_embed.proj.*", "blocks.<i>.*", "norm.*", "head.*");
 * parseq_forward* ignore decode_ar / refine_iters and return vitstr/system.py:65-71: head(norm(x))[:, 1 : max_length+2]
 * as logits [N, num_steps, num_tokens-2]; parseq_encode returns forward_features [N, T+1, D]. */
int parseq_create(const parseq_config* cfg, parseq_engine** out);
void parseq_destroy(parseq_engine* e);

/* Replaces model.PARSeq.load_state_dict as used by strhub/models/utils.py:80-82: `key` is a
 * state_dict key of the inner model (e.g. "encoder.blocks.3.attn.qkv.weight",
 * "decoder.layers.0.cross_attn.in_proj_weight", "pos_queries"); `data` is a HOST pointer to `numel`
 * contiguous fp32 values in PyTorch layout.  GEMM weight matrices are rounded to bf16 on upload. */
int parseq_set_weight(parseq_engine* e, const char* key, const float* data, int64_t numel);
/* Number of state_dict keys the engine expects, and the i-th key / its element count. */
int parseq_num_weights(const parseq_engine* e);
const char* parseq_weight_key(const parseq_engine* e, int i, int64_t* numel);

/* Input-independent precomputation (content K/V table over (position, token), query projections
 * of pos_queries); must be called after all weights are set and after any weight update. */
int parseq_finalize(parseq_engine* e, parseq_stream_t stream);

/* Decode options of one forward call: model.PARSeq.forward(tokenizer, images, max_length)
 * (model.py:105-169) with the module attributes decode_ar / refine_iters (model.py:55-56). */
typedef struct parseq_forward_args {
  int32_t batch;                         /* N images */
  int32_t max_length;                    /* -1 = None ("testing": early-exit length reported in *steps) */
  int32_t decode_ar;                     /* 0 / 1 */
  int32_t refine_iters;
  /* Optional teacher forcing (debug / parity): device int32 [batch, num_steps]; AR step i feeds
   * forced_ids[:, i+1] instead of its own argmax.  NULL in production. */
  const int32_t* forced_ids;
  /* Optional: device int32 [refine_iters, batch, num_steps] contexts (BOS included) for the cloze passes. */
  const int32_t* forced_refine;
  /* Optional per-image character allowlist: uint32 [batch][ceil(C / 32)] words, C = num_tokens - 2; bit c % 32 of word
   * c / 32 of row b allows class c for image b.  The result is that of the reference with its character head wrapped as
   * head(x)[b, :, c] = -inf for every disallowed c: every greedy decision (AR feedback, refine contexts, ids, the step
   * count S) is the argmax of the masked row, a disallowed class never wins (not even with a NaN or +inf raw logit),
   * and the returned logits hold exactly -inf there.  EOS (class 0) is always allowed, so an empty row decodes to the
   * empty label; an all-ones row gives the bits of an unmasked call.  NULL = no constraint, and no extra copy or
   * launch.  Same memory as the entry point's images: DEVICE for parseq_forward / _u8 / _crops, HOST for
   * the *_host* variants (uploaded with each super-chunk).  PARSeq and ViTSTR; not with forced_ids / forced_refine. */
  const uint32_t* class_mask;
  /* Optional output: fp32 [batch][num_steps][T] cross-attention maps, T = (img_h / patch_h) * (img_w / patch_w) image
   * tokens in the patch-embed flatten order (row-major over the patch grid).  maps[b][i][t] is ca_weights of the query
   * stream of the last decoder layer (strhub/models/parseq/modules.py:74, nn.MultiheadAttention's head average) in the
   * pass that produced logits[b][i]: the last cloze refinement pass (refine_iters >= 1), the NAR pass (decode_ar = 0), or
   * AR step i's query (decode_ar = 1, no refinement; computed by one teacher-forced pass over the AR loop's own ids [BOS,
   * ids[:, :num_steps-1]] under the causal masks, so it is the same whichever AR loop ran).  Rows follow the allowlist's
   * ids; rows past the early-exit length S are computed and may be dropped with the logits.  The logits, ids and steps
   * are bit-identical to the call without maps.  Same memory as the entry point's logits: DEVICE for parseq_forward /
   * _u8 / _crops, HOST for the *_host* variants.  NULL = no maps, no extra launch or allocation; the first call with maps
   * allocates a static [max_batch][max_label_length + 1][T] buffer (the first AR-only one also the causal masks of its
   * map pass, uploaded synchronously, so make it outside a stream capture).  PARSeq only (ViTSTR: PARSEQ_ERR_UNSUPPORTED); not
   * with forced_ids / forced_refine (PARSEQ_ERR_INVALID_ARG). */
  float* attn_maps;
} parseq_forward_args;

/* Replaces system.PARSeq.forward -> model.PARSeq.forward (system.py:87-88, model.py:105-169).
 *   images : DEVICE fp32 [N,3,H,W] (NCHW, values as produced by T.Normalize(0.5,0.5))
 *   logits : DEVICE fp32 [N, num_steps, num_tokens-2], num_steps = min(max_length, max_label_length)+1
 *            (max_label_length+1 if -1)
 *   ids    : DEVICE int32 [N, num_steps] argmax of `logits` (may be NULL)
 *   steps  : DEVICE int32 [1] (may be NULL): S = number of AR steps the reference would have run
 *            before its batch-wide early exit (model.py:144); == num_steps when max_length >= 0,
 *            when decode_ar == 0.  Only affects the returned SHAPE when refine_iters == 0. */
int parseq_forward(parseq_engine* e, const parseq_forward_args* args, const float* images,
                   float* logits, int32_t* ids, int32_t* steps, parseq_stream_t stream);

/* End-to-end variant with HOST buffers (pinned or pageable): H2D of images, forward, D2H of
 * logits / ids / steps, synchronised on return.  This is what bench.py times as `e2e`. */
int parseq_forward_host(parseq_engine* e, const parseq_forward_args* args, const float* images_host,
                        float* logits_host, int32_t* ids_host, int32_t* steps_host,
                        parseq_stream_t stream);

/* "Next" rows of the path (SURVEY.md section 8f).
 * Raw-crop input: images uint8 [N, H, W, 3] (HWC, as PIL / numpy hold them, already resized to img_size); the reference's
 * T.ToTensor() + T.Normalize(0.5, 0.5) (strhub/data/module.py:68-82) is folded into the patch gather.  Device / host
 * variants mirror parseq_forward / parseq_forward_host. */
int parseq_forward_u8(parseq_engine* e, const parseq_forward_args* args, const uint8_t* images_hwc,
                      float* logits, int32_t* ids, int32_t* steps, parseq_stream_t stream);
int parseq_forward_host_u8(parseq_engine* e, const parseq_forward_args* args, const uint8_t* images_hwc_host,
                           float* logits_host, int32_t* ids_host, int32_t* steps_host, parseq_stream_t stream);
/* Raw crops of any size: the whole reference transform (strhub/data/module.py:69-82: Image.rotate(rotation, expand=True),
 * T.Resize(img_size, BICUBIC) of the uint8 RGB image, ToTensor, Normalize(0.5, 0.5)) runs on the device.  The resize is
 * byte-identical to PIL's; the results are bit-identical to parseq_forward_u8 on the PIL-resized crops.  Each
 * super-chunk of max_batch crops is resized into the engine's static uint8 input, in front of the CUDA graph.  The only
 * device memory that grows with the crops is the staging copy of a super-chunk's bytes in the host variant. */
typedef struct parseq_crops {
  const uint8_t* data;     /* packed HWC RGB bytes of all crops: DEVICE (forward_crops, resize_crops) or HOST (forward_host_crops) */
  int64_t data_bytes;
  const int64_t* offsets;  /* HOST int64 [N]: byte offset of crop i in data */
  const int32_t* sizes;    /* HOST int32 [N][2]: (h, w) of crop i before rotation, 1 <= h, w <= 8192 */
  int32_t rotation;        /* 0, 90, 180, 270: PIL Image.rotate(r, expand=True), counter-clockwise */
  const int32_t* rotations;  /* HOST int32 [N]: crop i's own rotation (each 0, 90, 180 or 270), or NULL: `rotation` for
                                every crop.  A row's results do not depend on the other crops of the call, so crop i
                                reads exactly as in a call with rotation = rotations[i]. */
} parseq_crops;
/* out_hwc: DEVICE uint8 [N, img_h, img_w, 3], what T.Resize(img_size, BICUBIC) makes of each (rotated) crop.  The
 * metadata is checked on the host before anything is launched (PARSEQ_ERR_INVALID_ARG). */
int parseq_resize_crops(parseq_engine* e, int32_t batch, const parseq_crops* crops, uint8_t* out_hwc, parseq_stream_t stream);
/* Text regions of full frames (a detector's quadrilaterals) -> rectified crops that every raw-crop entry point takes.
 * Region i is crop size (h_i, w_i) and the 8 coefficients a0..a7 of PIL's PERSPECTIVE transform, which map output
 * point (u, v) to frame point x = (a0 u + a1 v + a2) / (a6 u + a7 v + 1), y = (a3 u + a4 v + a5) / (a6 u + a7 v + 1).
 * Its bytes are exactly frame.transform((w, h), Image.Transform.PERSPECTIVE, coeffs, Image.Resampling.BICUBIC) of the
 * RGB frame (Pillow's Geometry.c): per output pixel (x, y) the point (x + .5, y + .5) is mapped in fp64 in that order;
 * a point outside [0, W) x [0, H) gives 0; otherwise the 4 x 4 BICUBIC of Geometry.c (rows first, taps clamped to the
 * frame) gives v, written as 0 if v <= 0, 255 if v >= 255, else (uint8)v (truncation).  For a quadrilateral TL, TR, BR,
 * BL the Python layer derives (h, w) and the coefficients (Heckbert's square-to-quad map, parseq_b200/regions.py); an
 * integer box gives a = (1, 0, x0, 0, 1, y0, 0, 0), the crop frame[y0:y1, x0:x1] with 0 outside the frame.
 * One kernel thread per output pixel; a crop's bytes depend only on its own frame, size and coefficients. */
typedef struct parseq_regions {
  const uint8_t* frames;         /* DEVICE packed HWC RGB bytes of all frames */
  int64_t frames_bytes;
  const int64_t* frame_offsets;  /* HOST int64 [F]: byte offset of frame f in frames */
  const int32_t* frame_sizes;    /* HOST int32 [F][2]: (H, W) of frame f, 1 <= H, W <= 32768 */
  int32_t num_frames;            /* F */
  const int32_t* frame_index;    /* HOST int32 [M]: the frame of region i */
  const int32_t* sizes;          /* HOST int32 [M][2]: (h, w) of crop i, 1 <= h, w <= 8192 */
  const double* coeffs;          /* HOST double [M][8]: PIL PERSPECTIVE order, output (x + .5, y + .5) -> frame */
} parseq_regions;
/* out: DEVICE uint8, the M crops [h_i, w_i, 3] back to back (crop i at byte sum_{j<i} 3 h_j w_j), out_bytes at least
 * that sum.  Checked on the host before anything is enqueued, also without a handle (PARSEQ_ERR_INVALID_ARG): null
 * pointers, count < 0, frame sides outside [1, 32768] or frame bytes past frames_bytes, frame_index out of range, crop
 * sides outside [1, 8192], non-finite coefficients, a denominator a6 x + a7 y + 1 that is not positive at one of the
 * four corner pixel centres (then it is positive at every pixel centre), and out_bytes too small.  The region table is
 * uploaded per chunk of max_batch regions; the call runs on the engine's main stream, ordered after the caller's
 * earlier work on `stream`, and needs no weights. */
int parseq_warp_regions(parseq_engine* e, int32_t count, const parseq_regions* regions, uint8_t* out, int64_t out_bytes,
                        parseq_stream_t stream);
/* Curved text regions: polygons of F = 2k points, 3 <= k <= 32, in frame pixels (pixel i covers [i, i + 1)), rectified
 * by the thin-plate spline of TRBA's GridGenerator (RARE) with the polygon as its fiducial points C'.  The callers'
 * Total-Text / CTW1500 order (top edge p_0..p_{k-1} left to right, then bottom edge q_0..q_{k-1} right to left) becomes
 * the engine order C'_j = p_j, C'_{k+j} = b_j = q_{k-1-j} in Python; the C ABI takes the engine order.
 *   Crop size (the Python layer): w = max(1, floor(max(sum |p_{j+1} - p_j|, sum |b_{j+1} - b_j|) + 0.5)),
 *   h = max(1, floor(max_j |p_j - b_j| + 0.5)); with k = 2 this is the quad rule.
 *   Map, fp64: C_x = numpy.linspace(-1, 1, k) bit for bit, C_y = -1 (top) / +1 (bottom); T = inv_delta_C . [C'; 0]
 *   (parseq_tps_coeffs); output pixel (x, y) has xn = (2x + 1 - w) / w, yn = (2y + 1 - h) / h, r_m = |(xn, yn) - C_m|,
 *   phi_m = (r_m r_m) ln(r_m + 1e-6), and goes to X = T0 + T1 xn + T2 yn + sum_m T_{3+m} phi_m (that order, one rounding
 *   per operation, no FMA), Y likewise; (X, Y) then goes through parseq_warp_regions' sampler unchanged.
 *   Exactness: every operation is IEEE round-to-nearest except ln, which the device does not round as numpy does.  The
 *   bytes equal an fp64 restatement with numpy's log (tests/tps_warp_oracle.py) except at pixels whose byte changes when
 *   the mapped point moves by 1e-7 px; they are not PIL-exact as the quad warp is. */
typedef struct parseq_polygons {
  const uint8_t* frames;         /* DEVICE packed HWC RGB bytes of all frames */
  int64_t frames_bytes;
  const int64_t* frame_offsets;  /* HOST int64 [F]: byte offset of frame f in frames */
  const int32_t* frame_sizes;    /* HOST int32 [F][2]: (H, W) of frame f, 1 <= H, W <= 32768 */
  int32_t num_frames;            /* F */
  const int32_t* frame_index;    /* HOST int32 [M]: the frame of region i */
  const int32_t* sizes;          /* HOST int32 [M][2]: (h, w) of crop i, 1 <= h, w <= 8192 */
  const int32_t* num_points;     /* HOST int32 [M]: 2k_i points of region i, even, 6..64 (k may differ per region) */
  const double* points;          /* HOST double: the regions' points (x, y) back to back, engine order */
} parseq_polygons;
/* coeffs [F + 3][2] = T of the map above for the F = num_points points [F][2] (engine order): the host solve the warp
 * uses, with inv_delta_C computed once per k (Gauss-Jordan with partial pivoting, fp64, thread-safe cache).  No handle
 * or device.  PARSEQ_ERR_INVALID_ARG for null pointers, a count that is odd or outside [6, 64], non-finite points. */
int parseq_tps_coeffs(int32_t num_points, const double* points, double* coeffs);
/* out: DEVICE uint8, the M crops [h_i, w_i, 3] back to back (crop i at byte sum_{j<i} 3 h_j w_j), out_bytes at least
 * that sum.  Checked on the host before anything is enqueued, also without a handle (PARSEQ_ERR_INVALID_ARG): null
 * pointers, count < 0, the frame checks of parseq_warp_regions, frame_index out of range, crop sides outside [1, 8192],
 * point counts odd or outside [6, 64], non-finite points, and out_bytes too small.  Per chunk of max_batch regions the
 * coefficients are solved on the host and the table (descriptor, T and C_x per region) uploaded; region_tps_kernel runs
 * on the engine's main stream, ordered after the caller's earlier work on `stream`, and needs no weights. */
int parseq_warp_polygons(parseq_engine* e, int32_t count, const parseq_polygons* polygons, uint8_t* out,
                         int64_t out_bytes, parseq_stream_t stream);
/* parseq_forward_u8 / parseq_forward_host_u8 on the resized crops; args->batch = N.  No teacher forcing.  The host
 * variant uploads each super-chunk's bytes on the engine's copy stream (in two halves from 256 crops up, PARSeq). */
int parseq_forward_crops(parseq_engine* e, const parseq_forward_args* args, const parseq_crops* crops, float* logits,
                         int32_t* ids, int32_t* steps, parseq_stream_t stream);
int parseq_forward_host_crops(parseq_engine* e, const parseq_forward_args* args, const parseq_crops* crops,
                              float* logits_host, int32_t* ids_host, int32_t* steps_host, parseq_stream_t stream);
/* Orientation search: each crop read in the orientation the model is most confident of.
 * Rule.  The caller lists orientations o_0 .. o_{R-1} (1 <= R <= 4, distinct, each 0, 90, 180 or 270) and optionally a
 * threshold t (min_confidence; NaN = none).  Every crop is read at o_0; a crop whose confidence is >= t keeps that
 * reading.  Every other crop (every crop without t) is also read at o_1 .. o_{R-1} and takes the reading of highest
 * confidence; ties go to the earlier orientation of the list, and NaN ranks below every number.  A reading's confidence
 * is parseq_postprocess's, in its fp32 order: parseq_postprocess of the returned logits gives the returned confidence
 * bit for bit.  Each reading is bit-identical to parseq_forward_crops's at that rotation.
 * Schedule.  Pass 1 is parseq_forward_crops of all N crops at o_0, into the caller's outputs.  A confidence kernel then
 * writes o_0 and its confidence c_0 for every crop.  With t, c_0 is copied to the host, which lists the crops below t:
 * this is the call's one host synchronisation, so a call with t cannot be captured in a CUDA graph.  Pass 2 reads the
 * listed crops at the other R - 1 orientations: super-chunks of floor(max_batch / (R - 1)) crops, each crop's R - 1
 * readings in one super-chunk, the reading count rounded up to a power of two (at most max_batch) with copies of the
 * last reading, so a call adds graphs of power-of-two or max_batch readings only.  After each pass-2 super-chunk the
 * confidence kernel (one CTA per reading) scores every reading, and the orientation select kernel (one CTA per listed
 * crop, no atomics) compares a crop's readings and, when one wins, copies its logits, ids and maps into the crop's
 * outputs.
 * Outputs are those of parseq_forward_crops (DEVICE logits / ids / steps, attn_maps), plus rotation_out DEVICE int32 [N]
 * (the chosen orientation) and confidence_out DEVICE fp32 [N].  steps is the maximum over both passes.  Where the steps
 * shape the result (max_length = -1, decode_ar, refine_iters = 0, PARSeq), the rows of a crop's logits, ids and maps
 * from the step count of the pass (pass 2: of the super-chunk) that produced its reading are 0: they lie after that
 * reading's EOS.  crops->data may be device or host memory: host crops are staged per super-chunk, so the staging
 * buffer holds at most max_batch crops of pass 1 or the floor(max_batch / (R - 1)) largest crops; crops->rotations must
 * be NULL.  class_mask (DEVICE rows) and attn_maps as in parseq_forward_crops; each pass-2 reading uses its crop's mask
 * row.  Every argument is checked on the host before anything is enqueued (PARSEQ_ERR_INVALID_ARG; the orientations and
 * outputs also without a handle); max_batch must be >= R - 1. */
typedef struct parseq_orient_args {
  int32_t num_orientations;   /* R, 1..4 */
  int32_t orientations[4];    /* o_0 .. o_{R-1} */
  float min_confidence;       /* t, or NaN for none */
  int32_t* rotation_out;      /* DEVICE int32 [N] */
  float* confidence_out;      /* DEVICE fp32 [N] */
} parseq_orient_args;
int parseq_forward_crops_oriented(parseq_engine* e, const parseq_forward_args* args, const parseq_crops* crops,
                                  const parseq_orient_args* orient, float* logits, int32_t* ids, int32_t* steps,
                                  parseq_stream_t stream);
/* Candidate scoring: the log-likelihood of given labels for each image, e.g. to pick the best word of a lexicon.
 * PARSeq: score(x, c) = sum_{i=0..n} log_softmax(head(decode(tgt_in, memory, content_mask, query_mask)))[i, t_i] with
 * tgt_in = [BOS, c_1..c_n] (Tokenizer.encode, strhub/data/utils.py:113-118, without its last column), the targets
 * t = (c_1..c_n, EOS) and the masks of the canonical left-to-right permutation (generate_attn_masks,
 * strhub/models/parseq/system.py:153-167): minus the summed cross-entropy terms of permutation 0 of training_step
 * (system.py:169-197).  ViTSTR: sum_{i=0..n} log_softmax(head(norm(x))[:, 1:])[i, t_i], minus the summed terms of
 * CrossEntropySystem.forward_logits_loss (strhub/models/base.py:194-201).  Each term equals torch.log_softmax(row, -1)[t]
 * of the fp32 logits row up to fp32 rounding (a row holding NaN or +inf gives NaN); the logits never reach memory.  The
 * encoder runs once per image, the decoder once per candidate over its n + 1 positions.  Runs eagerly (no CUDA graph);
 * the first call allocates the scoring buffers. */
typedef struct parseq_score_args {
  int32_t batch;               /* N images */
  int32_t num_candidates;      /* M = sum of per_image */
  const int32_t* per_image;    /* HOST int32 [N]: candidates of image b, >= 1; candidates are image-major */
  const int32_t* targets;      /* HOST int32 [M][max_label_length + 1]: c_1..c_n (head classes 1..C-1), EOS (0), rest ignored */
  const int32_t* lengths;      /* HOST int32 [M]: n, 0 <= n <= max_label_length */
  float* attn_maps;            /* DEVICE fp32 [M][max_label_length + 1][T] or NULL: see below */
} parseq_score_args;
/* images as parseq_forward / parseq_forward_u8 take them; scores DEVICE fp32 [M]; token_logprobs DEVICE fp32
 * [M][max_label_length + 1] or NULL (term i of candidate m, 0 past n).  All metadata is checked on the host before anything
 * is launched (PARSEQ_ERR_INVALID_ARG): the counts need no handle, the targets are checked against the handle's
 * configuration (ids, EOS at position n and nowhere before, no BOS / PAD). */
int parseq_score(parseq_engine* e, const parseq_score_args* a, const float* images, float* scores, float* token_logprobs,
                 parseq_stream_t stream);
int parseq_score_u8(parseq_engine* e, const parseq_score_args* a, const uint8_t* images_hwc, float* scores,
                    float* token_logprobs, parseq_stream_t stream);
/* attn_maps (PARSeq; ViTSTR has no decoder cross-attention: PARSEQ_ERR_UNSUPPORTED): row i <= n of candidate m is the
 * cross-attention of the decoder's last layer for the query that predicts t_i in the teacher-forced pass above (the
 * head-averaged weights nn.MultiheadAttention returns, as parseq_forward_args.attn_maps), rows past n are 0.  The maps are
 * written in the pass that computes the scores, which stay bit-identical to the call without maps; a row's bits do not
 * depend on the other candidates of its image or on the batch.  No buffer is allocated for them. */
/* The host checks of parseq_score against a configuration, without a handle or a device. */
int parseq_score_check(const parseq_config* cfg, const parseq_score_args* a);

/* Beam search: the K most likely readings of each image with their log-likelihoods (the quantity parseq_score computes).
 * One search per image, beam width K, over num_steps = min(max_length, max_label_length) + 1 positions:
 *   - K slots per image; slot 0 starts as [BOS] with score 0, the others empty (score -inf).
 *   - Step i: every active slot runs the AR step at query position i over its own prefix (model.py:124-142 for one row).
 *     Over the allowed classes of its logits row, LSE = log-sum-exp (NaN if one is NaN or +inf); a class's term is logit - LSE (fp32) and a child's
 *     score is parent + term.  The slot expands its K best classes in the row order: NaN logits first (lowest class
 *     first), then logit descending, ties to the lower class.  Classes the allowlist masks or whose logit is -inf never
 *     expand.
 *   - A child that takes EOS is finished with its length n; one that reaches num_steps characters without EOS is finished
 *     with num_steps characters.  A finished slot is carried unchanged into every later pool.
 *   - The pool, in slot order, holds each finished slot and each active slot's expansions in row order; the K best by
 *     score are kept by a stable sort (NaN after every number; -inf never kept).  They are the next step's slots.
 * PARSeq runs the AR decoder whatever decode_ar / refine_iters say and never refines; ViTSTR applies the same rule to its
 * per-position logits head(norm(x))[:, 1:] (the row of step i is the image's position-i row for every slot).  With K = 1
 * the ids through the first EOS are the greedy AR ids.  Runs eagerly (no CUDA graph); the first call allocates the beam
 * buffers.  Arguments are checked on the host before anything is launched (PARSEQ_ERR_INVALID_ARG). */
typedef struct parseq_beam_args {
  int32_t batch, beam_width, max_length;   /* 1 <= beam_width <= 16 (PARSeq: and <= option dec_chunk); max_length -1 = None */
  const uint32_t* class_mask;              /* DEVICE allowlist rows as parseq_forward_args.class_mask, or NULL */
  float* attn_maps;                        /* DEVICE fp32 [N][K][num_steps][T] or NULL: see below */
} parseq_beam_args;
/* images as parseq_forward / parseq_forward_u8 take them; all outputs DEVICE, hypotheses best first:
 * ids int32 [N][K][num_steps] = c_1..c_n, then 0 (EOS / padding); lengths int32 [N][K] = n, -1 for a missing hypothesis;
 * scores fp32 [N][K], -inf for a missing hypothesis (e.g. allowlist "": the only reading is "" with score 0).
 * attn_maps (PARSeq, also under a lexicon; ViTSTR: PARSEQ_ERR_UNSUPPORTED): row i <= n of hypothesis k is the
 * cross-attention map parseq_score_args.attn_maps gives row i of that hypothesis's label, bit for bit; rows past n, and
 * every row of a missing hypothesis, are 0.  After a group's last selection one teacher-forced pass over its final
 * hypotheses (context [BOS, c_1..c_{num_steps-1}] under the causal masks) computes them on the device; the ids, lengths
 * and scores are bit-identical to the call without maps. */
int parseq_beam_search(parseq_engine* e, const parseq_beam_args* a, const float* images, int32_t* ids, int32_t* lengths,
                       float* scores, parseq_stream_t stream);
int parseq_beam_search_u8(parseq_engine* e, const parseq_beam_args* a, const uint8_t* images_hwc, int32_t* ids,
                          int32_t* lengths, float* scores, parseq_stream_t stream);

/* Lexicon-constrained beam search: every hypothesis is a word of a lexicon, at a cost that depends on the beam width and
 * not on the lexicon's size.  A lexicon is a set of words over the head classes 1..C-1, compiled to a rooted DAG in
 * topological numbering (a trie is one): nodes 0..V-1, terminal[v] != 0 when the path from a root to v spells a word, and
 * the edges of node v at first_edge[v] .. first_edge[v+1]-1, each with a head class edge_class (1..C-1, strictly
 * increasing within a node) and a child edge_child (> v).  Image b starts at node roots[b].
 * The rule is parseq_beam_search's, except that each slot also carries its node v.  At step i an active slot
 *   - takes its LSE exactly as there: over the allowlist-allowed classes of the whole row, not over v's children (the
 *     lexicon restricts the hypotheses, it does not renormalise the model);
 *   - may expand EOS iff terminal[v], and each edge class c of v iff the allowlist allows c, logit[c] != -inf and
 *     i + 1 < num_steps (a character leaves room for its EOS);
 *   - expands its K best expandable classes in the row order; a character moves the child to edge_child, EOS finishes it
 *     with length i.
 * The pool, the stable sort, NaN ranking and -inf handling are unchanged.  So every hypothesis is a word of at most
 * num_steps - 1 characters that ended with EOS, and its score is parseq_score's for that word; with K >= the number of
 * words and no allowlist or -inf pruning the search is exhaustive (distinct prefixes of one length are distinct words). */
typedef struct parseq_lexicon parseq_lexicon;   /* a lexicon on an engine's device (parseq_lexicon_create) */
typedef struct parseq_lexicon_desc {
  int32_t num_nodes, num_edges;   /* V >= 1, E >= 0 (E = 0: the lexicon {""}) */
  const int32_t* first_edge;      /* HOST int32 [V + 1], non-decreasing, first_edge[0] = 0, first_edge[V] = E */
  const int32_t* edge_class;      /* HOST int32 [E] */
  const int32_t* edge_child;      /* HOST int32 [E] */
  const uint8_t* terminal;        /* HOST uint8 [V], nonzero where the node ends a word */
} parseq_lexicon_desc;
/* The host checks of a lexicon against a configuration, without a handle or a device (PARSEQ_ERR_INVALID_ARG): counts,
 * first_edge monotone and ending at E, classes in 1..C-1 and strictly increasing within a node, children in v+1..V-1, and
 * no path longer than max_label_length edges. */
int parseq_lexicon_check(const parseq_config* cfg, const parseq_lexicon_desc* d);
/* Checks the lexicon against the engine's configuration, then uploads it to the engine's device on `stream` (the call
 * returns once the copy is done; the host arrays are not kept).  The handle may serve any engine on that device with the
 * same number of classes, and outlives the engine it was made with. */
int parseq_lexicon_create(parseq_engine* e, const parseq_lexicon_desc* d, parseq_lexicon** out, parseq_stream_t stream);
void parseq_lexicon_destroy(parseq_lexicon* lx);
/* parseq_beam_search under a lexicon; `roots` HOST int32 [batch] (each in 0..V-1; pageable or pinned, copied before the
 * call returns, so the buffer may be reused at once) or NULL for node 0 everywhere.  Outputs as parseq_beam_search.  Checked on the host before anything is launched: the lexicon is
 * on the engine's device with the engine's number of classes, and every root is a node.  The first lexicon call allocates
 * the lexicon's beam state (a node per beam row, double-buffered) and, above 128 classes, one fp32 logits buffer per stage:
 * the lexicon step reads the chain's logits rows rather than the top-K epilogue's keys, whose classes need not be
 * children of the slot's node. */
int parseq_beam_search_lexicon(parseq_engine* e, const parseq_beam_args* a, const parseq_lexicon* lx, const int32_t* roots,
                               const float* images, int32_t* ids, int32_t* lengths, float* scores, parseq_stream_t stream);
int parseq_beam_search_lexicon_u8(parseq_engine* e, const parseq_beam_args* a, const parseq_lexicon* lx,
                                  const int32_t* roots, const uint8_t* images_hwc, int32_t* ids, int32_t* lengths,
                                  float* scores, parseq_stream_t stream);

/* Fused post-processing of BaseSystem._eval_step (strhub/models/base.py:132-142) + Tokenizer._filter
 * (strhub/data/utils.py:120-129): DEVICE logits [N, num_steps, num_classes] -> ids [N, num_steps] (greedy), lengths [N]
 * (index of the first EOS, num_steps if none) and confidence [N] (product of the max softmax probabilities up to and
 * including the EOS position). */
int parseq_postprocess(const float* logits, int32_t batch, int32_t num_steps, int32_t num_classes, int32_t eos_id,
                       int32_t* ids, int32_t* lengths, float* confidence, parseq_stream_t stream);

/* Replaces model.PARSeq.encode (model.py:83-84): memory DEVICE fp32 [N, T, D]. */
int parseq_encode(parseq_engine* e, int32_t batch, const float* images, float* memory,
                  parseq_stream_t stream);

/* Replaces model.PARSeq.decode (strhub/models/parseq/model.py:86-103 -> modules.py:55-125): tgt DEVICE int32 [N, J] context ids (tgt[:, 0] = BOS; token k >= 1 receives pos_queries[k-1], model.py:96-99),
 * memory DEVICE fp32 [N, T, D] (what parseq_encode returns), query DEVICE fp32 [N, NQ, D] or NULL (= pos_queries[:NQ],
 * model.py:100-101), query_mask DEVICE uint8 [NQ, J] or NULL (1 = key masked for that query: the bool `tgt_query_mask`),
 * padding_mask DEVICE uint8 [N, J] or NULL (`tgt_padding_mask`); out DEVICE fp32 [N, NQ, D] = Decoder output including
 * the final LayerNorm (modules.py:123-125).  1 <= J, NQ <= max_label_length + 1.  A query whose keys are all masked
 * yields NaN, as the reference's softmax does.  Same as parseq_decode_ex with content_mask = NULL. */
int parseq_decode(parseq_engine* e, int32_t batch, int32_t ctx_len, int32_t num_queries, const int32_t* tgt,
                  const float* memory, const float* query, const uint8_t* query_mask, const uint8_t* padding_mask,
                  float* out, parseq_stream_t stream);
/* parseq_decode with the content-stream mask `tgt_mask`: content_mask DEVICE uint8 [J, J] or NULL (unmasked, as
 * tgt_mask=None is), 1 = key masked for that context row; the padding mask applies to the content rows too.  Decoders of
 * depth >= 2 update the content stream in every layer but the last (modules.py:117-123), so the mask acts there; at
 * depth 1 the content stream is never updated and the mask has no effect. */
int parseq_decode_ex(parseq_engine* e, int32_t batch, int32_t ctx_len, int32_t num_queries, const int32_t* tgt,
                     const float* memory, const float* query, const uint8_t* query_mask, const uint8_t* padding_mask,
                     const uint8_t* content_mask, float* out, parseq_stream_t stream);
/* Replaces model.PARSeq.head (model.py:63: nn.Linear(embed_dim, num_tokens - 2)): x DEVICE fp32 [rows, D] ->
 * logits DEVICE fp32 [rows, num_tokens - 2] (bf16 tensor-core operands, fp32 accumulate). */
int parseq_head(parseq_engine* e, int32_t rows, const float* x, float* logits, parseq_stream_t stream);
/* Replaces TokenEmbedding.forward (modules.py:175-176): out[i, :] = sqrt(D) * embedding[ids[i], :], DEVICE fp32 [n, D]. */
int parseq_text_embed(parseq_engine* e, int32_t n, const int32_t* ids, float* out, parseq_stream_t stream);

/* Introspection used by bench.py / tests. */
int64_t parseq_kernel_launches(const parseq_engine* e);      /* cumulative count of kernels launched */
/* Microbenchmark of the AR kernel's TMA ring (tests/bench_tma_stream.py): `ctas` CTAs in clusters of `cluster` stream `nboxes`
 * 16 KB boxes each from `buf` through `nslot` slots, no compute. */
int parseq_bench_tma_stream(void* buf, int64_t bytes, int cluster, int ctas, int nboxes, int nslot, int mode, void* sink,
                            parseq_stream_t stream);
/* Debug counters by name ("ar2_occupancy_mt2", "ar2_clusters_mt2", "ar_last_per", "ar_last_clusters", "sm_count"; the last
 * cluster AR kernel instantiation: "ar_last_cluster_size", "ar_last_mt", "ar_last_head_split", "ar_last_wide",
 * "ar_last_ids_pitch"; "ar_last_path": the AR loop of the last PARSeq forward, 0 the chain of separate kernels, 1 the
 * grid-barrier kernel, 2 the cluster kernel, -1 no AR loop; "ln_clusters": the clusters the persistent GEMM + LayerNorm
 * kernel runs on, 0 before its first launch, also with e = NULL for the bare kernel exports; "beam_bytes": device bytes of
 * the beam-search buffers, 0 until the first parseq_beam_search call; process-wide, also with e = NULL:
 * "live_device_bytes" and "live_cuda_objects", the device bytes and the streams, events and graph execs that every live
 * handle and lexicon holds); "orient_rereads": the crops pass 2 of the last parseq_forward_crops_oriented call re-read,
 * and "orient_readings": the readings it ran, padding included; -1 if unknown. */
int64_t parseq_debug_int(parseq_engine* e, const char* name);
/* Options: "max_batch" (images per super-chunk = one CUDA graph), "chunk" (images per encoder pass inside a
 * super-chunk), "dec_chunk" (images per decoder chain; the chains of a super-chunk run concurrently on their own
 * streams), "use_graph" (0/1), "pdl" (programmatic dependent launch, 0/1), "timing" (1: record a CUDA-event pair around every launch
 * for parseq_get_timing; 0: off + clear), "block_n" (accepted for compatibility: the GEMM has one 128 x 128 tile), "fuse_ln" (bit 0: the attention-projection GEMM, bit 1: the fc2 GEMM
 * also produces the LayerNorm that follows it, used when the batch fills the machine at least twice with 128-row tiles; bit 2:
 * for any batch; default 3; 0: separate LayerNorm kernels), "ar_kernel" (AR loop: 2 = cluster-owned persistent kernel,
 * default, where it applies - decoders of depth >= 2 run the chain; 1 = grid-barrier persistent kernel, at most 128 head classes, max_label_length <= 31 and dec_depth 1; 0 = chain of separate kernels), "fuse_mlp" (1: fc1 + GELU + fc2 + residual +
 * LayerNorm of an encoder block in one kernel where fuse_ln bit 1 applies - bit-identical results, default 0), "attn_impl"
 * (encoder attention: 0 = mma.sync kernels, default; 1 = wgmma kernel), "ln_cta_group" / "mlp_cta_group"
 * (0 auto, 1 single CTA, 2 CTA pair sharing the weight tiles by TMA multicast: fused GEMM+LayerNorm / one-kernel
 * MLP; "cta_group" is accepted for compatibility, the GEMM runs single-CTA tiles), "ln_split" (fused GEMM+LayerNorm: 0 auto = the persistent column-split CTA-pair kernel at D = 384,
 * 1 never = the full-row kernel (ln_cta_group picks its single-CTA or pair form), 2 always), "pair_pdl", "gemm_stages" (kernel-variant switches for tests).  Options are PER HANDLE; with
 * e == NULL the launch options (block_n, attn_impl, pdl, gemm_stages, cta_group, ln_cta_group, mlp_cta_group, ln_split,
 * pair_pdl) set the
 * process defaults that the stand-alone kernel
 * entry points below use and that handles created afterwards inherit. */
int parseq_set_option(parseq_engine* e, const char* name, int64_t value);
/* After a synchronised forward with "timing"=1: device milliseconds, algorithmic FLOPs and launch count of
 * category 0 encoder GEMM, 1 encoder attention, 2 LayerNorm, 3 decoder GEMM, 4 decoder attention, 5 other,
 * 6 encoder residual GEMM fused with LayerNorm, 7 persistent AR-loop kernel, 8 scoring tail (head GEMM with the log-sum-exp
 * epilogue and the per-candidate reduce of parseq_score), 9 beam selection (the selection kernel and, at dec_depth >= 2,
 * the K/V cache gather of parseq_beam_search), 10 cross-attention maps (the maps kernels of parseq_forward_args,
 * parseq_score_args and parseq_beam_args.attn_maps and the beam maps' tail fill; the teacher-forced map passes' other
 * kernels count in their own categories), 11 orientation search (the confidence and
 * select kernels and the pass-2 allowlist gather of parseq_forward_crops_oriented). */
int parseq_get_timing(parseq_engine* e, int category, double* ms, double* flops, int64_t* count);
/* Debug: after a forward with option "ar_prof"=1, copies the [32 steps][16 slots] globaltimer (ns) stamps that block 0 of
 * the persistent AR kernel recorded at its phase boundaries.  Row 26 holds extra stamps of step 1 of the cluster kernel;
 * with max_label_length > 31 only steps < 26 are recorded. */
int parseq_get_ar_profile(parseq_engine* e, uint64_t* out512);
const char* parseq_last_error(void);
const char* parseq_version(void);

/* Stand-alone kernel entry points (unit tests of the building blocks; all pointers DEVICE). */
/* C[M,N] = epilogue(A[M,K](bf16,row-major,lda) * W[N,K]^T(bf16,row-major,ldw) + bias) on wgmma.
 * mode: 0 -> fp32 out (alpha*(acc+bias) [+ resid[row % resid_mod or row]]), 1 -> bf16 out,
 *       2 -> bf16 gelu(acc+bias). */
int parseq_gemm_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, const float* bias,
                     int M, int N, int K, int mode, float alpha, const float* resid, int64_t ldr,
                     int resid_mod, void* out, int64_t ldo, parseq_stream_t stream);
/* Residual GEMM fused with the LayerNorm that follows it (timm Block: x = x + proj(attn) ; norm2(x) and
 * x = x + fc2(..) ; next norm1(x)):  x_inout[M, D] += A[M, K] * W[D, K]^T + bias (fp32, in place),
 * xn_bf16[M, D] = bf16(LayerNorm(x_inout; gamma, beta, eps)).  D in {192, 384}. */
int parseq_gemm_ln_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, const float* bias,
                        int M, int D, int K, float* x_inout, const float* gamma, const float* beta,
                        float eps, void* xn_bf16, parseq_stream_t stream);
/* The whole MLP of a timm Block + the LayerNorm that follows (x = x + fc2(GELU(fc1(norm2(x)))) ; next norm1(x)) in one
 * kernel: x_inout[M, D] += GELU(xn[M, D] * W1[4D, D]^T + b1) * W2[D, 4D]^T + b2 (fp32, in place; the bf16 hidden activation
 * stays on the SM), xn_out_bf16[M, D] = bf16(LayerNorm(x_inout; gamma, beta, eps)); xn_out_bf16 may alias xn.  D in {192, 384}. */
int parseq_mlp_ln_bf16(const void* xn, const void* W1, const float* b1, const void* W2, const float* b2,
                       int M, int D, float* x_inout, const float* gamma, const float* beta, float eps,
                       void* xn_out_bf16, parseq_stream_t stream);
/* y = bf16(LayerNorm(x; gamma, beta, eps)), x fp32 [M, D]. */
int parseq_layernorm_bf16(const float* x, const float* gamma, const float* beta, float eps, int M,
                          int D, void* y_bf16, float* y_f32_or_null, parseq_stream_t stream);
/* out[B*T, D] = softmax(QK^T/sqrt(64)) V per (image, head) from packed qkv bf16 [B*T, 3D]. */
int parseq_enc_attention(const void* qkv_bf16, int B, int T, int D, int heads, void* out_bf16,
                         parseq_stream_t stream);
/* The QKV projection and the attention core in one kernel: out[B*T, D] = softmax(QK^T/sqrt(64)) V per (image, head) with
 * [Q | K | V] = bf16(xn[B*T, D] * W_qkv[3D, D]^T + b_qkv) (b_qkv may be NULL); qkv never leaves the SM.  Bit-identical to
 * parseq_gemm_bf16 (mode 1) followed by parseq_enc_attention.  T = 128, D = 64 * heads in {192, 384}; anything else
 * returns PARSEQ_ERR_UNSUPPORTED. */
int parseq_qkv_attention_bf16(const void* xn_bf16, const void* W_qkv, const float* b_qkv, int B, int T, int D,
                              int heads, void* out_bf16, parseq_stream_t stream);
/* The head GEMM of parseq_score with its log-sum-exp epilogue: the logits v = A[M,K] * W[N,K]^T + bias (bias may be NULL)
 * never reach memory.  part: fp32 [M][ceil(N / 128)][2], per row and 128-column tile (max, sum of exp(v - max)) over the
 * tile's columns < N (a tile whose max is -inf sums exp(v)); tlogit[r] = v[r][tgt[r]] for tgt[r] in 0..N-1 (tgt and
 * tlogit both NULL: partials only).  Rows >= M are not written. */
int parseq_head_lse_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, const float* bias, int M, int N, int K,
                         const int32_t* tgt, float* part, float* tlogit, parseq_stream_t stream);
/* The head GEMM of parseq_beam_search above 128 classes with its top-K epilogue: part as parseq_head_lse_bf16 over the
 * allowed classes (a masked class counts as -inf), and keys: uint64 [M][ceil(N / 128)][16], the tile's k best allowed
 * classes in the beam order (see parseq_beam_select), 0 after the last; -inf logits are never listed.  1 <= k <= 16.
 * mask: allowlist words (parseq_forward_args.class_mask), row r reads row r / mask_div (mask_div >= 1), or NULL. */
int parseq_head_topk_bf16(const void* A, int64_t lda, const void* W, int64_t ldw, const float* bias, int M, int N, int K,
                          int k, const uint32_t* mask, int mask_div, float* part, uint64_t* keys, parseq_stream_t stream);
/* One step of parseq_beam_search's selection for `batch` images (one launch of the selection kernel).  An image's state
 * has one row r = b * beam_width + k per slot: ids [rows][ids_ld] (BOS, c_1.., then anything), score, len (characters, -1
 * empty) and st (0 active, 1 finished, 2 empty).  The logits row of slot (b, k) is row0 + b * img_stride + k *
 * slot_stride; it is read from `logits` [rows][num_classes], or, when keys != NULL and there is no lexicon, from the
 * partials and keys of parseq_head_topk_bf16 (part [rows][ntiles][2], keys [rows][ntiles][16], k = beam_width).  A key
 * orders a row's classes: NaN logits first, then the logit descending, ties to the lower class, -0 as +0.  The new
 * state goes to the *_out arrays, parent[r] = the state row slot r came from; at the last step (step + 1 == num_steps)
 * also out_ids [rows][num_steps], out_len [rows] and out_score [rows] as parseq_beam_search returns them.  With
 * first_edge != NULL the step walks a lexicon DAG (parseq_lexicon_desc arrays on the device; roots [batch] or NULL for
 * node 0, read at step 0; node_in read at step > 0; node_out written).  All pointers DEVICE.  Checked on the host
 * (PARSEQ_ERR_INVALID_ARG, nothing launched): 1 <= beam_width <= 16, ntiles == ceil(num_classes / 128), 0 <= step <
 * num_steps, ids_ld > num_steps, and logits present without keys or with a lexicon. */
typedef struct parseq_beam_select_args {
  const float* logits;                   /* [rows][num_classes] or NULL */
  const float* part;                     /* [rows][ntiles][2] or NULL */
  const uint64_t* keys;                  /* [rows][ntiles][16] or NULL */
  int32_t ntiles;
  int64_t row0, img_stride, slot_stride;
  int32_t batch, num_classes, beam_width, step, num_steps;
  const uint32_t* class_mask;            /* [batch][mask_ld] or NULL */
  int32_t mask_ld;
  const int32_t* ids_in;
  const float* score_in;
  const int32_t* len_in;
  const int32_t* st_in;
  int32_t* ids_out;
  float* score_out;
  int32_t* len_out;
  int32_t* st_out;
  int32_t* parent;
  int32_t ids_ld;
  int32_t* out_ids;
  int32_t* out_len;
  float* out_score;
  const int32_t* first_edge;             /* lexicon, or NULL */
  const int32_t* edge_class;
  const int32_t* edge_child;
  const uint8_t* terminal;
  const int32_t* roots;
  const int32_t* node_in;
  int32_t* node_out;
} parseq_beam_select_args;
int parseq_beam_select(const parseq_beam_select_args* a, parseq_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* PARSEQ_B200_H_ */
