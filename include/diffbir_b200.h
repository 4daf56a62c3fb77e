/* diffbir_b200 — C ABI of libdiffbir_b200.so (hand-written sm_90a kernels).
 *
 * This is the drop-in boundary for the DiffBIR restoration hot path. The reference
 * (XPixelGroup/DiffBIR) has no FFI: every op below replaces a PyTorch library call made
 * from the reference's nn.Module.forward methods; each entry cites the reference
 * file:line it stands in for (paths relative to the reference checkout).
 *
 * Conventions
 *  - All pointers are DEVICE pointers owned by the caller (PyTorch allocations); the
 *    library never allocates or frees device memory and only enqueues work on `stream`
 *    (a cudaStream_t passed as void*), so every call is CUDA-graph capturable.
 *  - Return value: 0 on success, < 0 on error; dbir_last_error() returns a thread-local
 *    message. No C++ exceptions cross the boundary.
 *  - "op16" is the 16-bit tensor-core operand format reported by dbir_operand_kind()
 *    (1 = IEEE fp16, 0 = bf16). Activations are NHWC; residual streams are fp32.
 */
#ifndef DIFFBIR_B200_H
#define DIFFBIR_B200_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif

/* ---- library info ------------------------------------------------------------------ */
const char* dbir_version(void);
const char* dbir_last_error(void);
int dbir_operand_kind(void);          /* 1 = fp16 operands, 0 = bf16 operands */
int dbir_sm_count(void);              /* SMs of the current device (cached) */

/* ---- wgmma GEMM / implicit 3x3 convolution --------------------------------------
 * out = residual + alpha * act(A * B^T + bias + rowvec)          (GEGLU: a * gelu(g))
 * Replaces nn.Linear (attention.py:22,35-42,67-73,310,331; swinir.py:21-31,104,106),
 * nn.Conv2d 3x3 / 1x1 (unet.py:67,99,149-153,173-188; controlnet.py:309-312;
 * vae.py:24-27,77-95,241-252,445-447,520-522; swinir.py:472,700-705,790-811) and the
 * elementwise adds around them (unet.py:216-223, attention.py:265-274,353,
 * controlnet.py:36-43, cldm.py:164).
 */
typedef struct dbir_gemm_args {
  const void* a;        /* op16. a_mode 0: [M, lda]; a_mode 1: NHWC [img_n, img_h, img_w, img_c] */
  const void* b;        /* op16 packed weight [N, ldb], K contiguous (conv: k = tap*C + c) */
  void* out;            /* fp32 or op16 [rows, ldo] */
  const float* bias;    /* [N] or NULL */
  const float* rowvec;  /* [M / rows_per_vec, N] added per row group (time embedding) or NULL */
  const float* residual;/* fp32 [rows, ldr] or NULL */
  int64_t lda, ldb, ldo, ldr;   /* element strides; lda/ldb 0 = K. a_mode 1: lda > 0 = pixel stride of `a` (>= img_c) */
  int32_t M, N, K;
  int32_t a_mode;       /* 0 plain matrix, 1 implicit conv (ksize x ksize, stride 1, pad ksize/2) */
  int32_t img_n, img_h, img_w, img_c, ksize;
  int32_t rows_per_vec; /* a_mode 0 only; conv mode uses the image index */
  int32_t out_kind;     /* 0 fp32, 1 op16 */
  int32_t act;          /* 0 none, 1 GELU(erf), 2 LeakyReLU(act_param), 3 SiLU, 4 quick_gelu x * sigmoid(1.702 x)
                           (CLIP MLP, clip_encoder.py -> CLIPMLP with hidden_act "quick_gelu") */
  int32_t geglu;        /* B rows packed per force_bn-row tile as [values | gates]; out has N/2 columns:
                           1 = values * gelu(gates) (GEGLU), 2 = values * silu(gates) (LLaMA's SwiGLU MLP,
                           down_proj(act(gate_proj(x)) * up_proj(x)) with values = up, gates = gate) */
  int32_t force_bn;     /* 0 = auto tile width, else 32/64/128/160/256 (required with geglu) */
  float alpha;          /* scale applied before the residual add (control strength) */
  float act_param;
  int32_t bias_per_row; /* 1: bias[row] instead of bias[col] (transposed products) */
  int32_t groups;       /* 0/1 = one problem. G > 1: G same-shape problems in one launch (e.g. the UNet and
                           ControlNet encoders' twin layers): A / out / residual / rowvec / gn_partials hold the G
                           problems back to back along M (M = total rows, divisible by G; conv: img_n divisible by
                           G), b is [G*N, ldb] and bias [G*N] (group g's weights at rows g*N). */
  void* splitk_ws;      /* optional split-K scratch (zero-initialised once by the caller, >= 64 KiB +
                           partial tiles); NULL disables split-K. Summation order is fixed. */
  int64_t splitk_ws_bytes;
  int32_t split_k;      /* 0 = auto, 1 = off, n > 1 = force n splits */
  int32_t cta_pair;     /* CTA pairs (2-CTA clusters sharing the B tile by TMA multicast): 0 = auto, 1 = whenever the tile count is even, 2 = never */
  void* gn_partials;    /* optional fp32 [img][dbir_gemm_gn_slots()][N][2]: per 32-row-slot column sums and
                           sums of squares of the OUTPUT (fused GroupNorm statistics; see dbir_gn_finalize) */
  int32_t gn_rows_per_img; /* matrix mode only: rows per image (multiple of 32); conv mode uses img_h*img_w */
} dbir_gemm_args;
/* Number of 32-row slots per image dbir_gemm writes into gn_partials (conv: h, w > 0; matrix: rows_per_img). */
int32_t dbir_gemm_gn_slots(int32_t conv_h, int32_t conv_w, int32_t rows_per_img);
int dbir_gemm(const dbir_gemm_args* args, void* stream);
/* dbir_gemm keeps a plan (tile width, CTA pairing, split-K) per problem signature. The first call
 * for a signature made outside stream capture times the candidate plans on the caller's operands
 * (outputs redirected to scratch, cold L2) and caches the fastest; DBIR_GEMM_AUTOTUNE=0 selects
 * the analytic model instead (bit-reproducible across processes: split-K changes summation order). */
/* the analytic model's plan for a tile grid, host only: out[0..3] = BN, splits, k-blocks per split, pair */
int dbir_gemm_model_plan(int32_t m_tiles, int32_t N, int32_t num_kb, int32_t geglu, int32_t force_bn,
                         int32_t split_k, int32_t cta_pair, int64_t ws_floats, int32_t* out);

/* ---- flash attention, head_dim 64 (wgmma) --------------------------------------------
 * out[b, i, h*64 + :] = softmax_j(q_h[i] . k_h[j] / 8) v_h[j]; q/k/v/out are op16 matrices
 * [batch, s, ld*] whose first heads*64 columns (from the given base pointer) hold the heads.
 * Replaces F.scaled_dot_product_attention and the head split/merge copies in
 * SDPCrossAttention.forward (attention.py:189-216); kv = text context for attn2.
 */
/* The optional workspace enables the stream-K decomposition: when whole 128-query tiles would
 * leave the last wave of CTA slots (two per SM) mostly idle, every CTA instead takes an equal share
 * of the (tile, 64-key step) space and tiles cut by a CTA boundary are combined through `ws` (fixed
 * part order: deterministic). ws: dbir_attention_ws_bytes() bytes, zero-initialised once by the
 * caller, private to one stream; NULL / too small = whole tiles per CTA. */
int dbir_attention(const void* q, const void* k, const void* v, void* out, int32_t batch,
                   int32_t heads, int32_t sq, int32_t skv, int64_t ldq, int64_t ldk, int64_t ldv,
                   int64_t ldo, void* ws, int64_t ws_bytes, void* stream);
int64_t dbir_attention_ws_bytes(int32_t batch, int32_t heads, int32_t sq, int32_t skv);  /* 0: not needed */

/* ---- GroupNorm (32 groups) / LayerNorm ------------------------------------------------
 * dbir_gn_stats: per-(image, group) mean and rstd of the virtual concat [src1 | src2] (fp32
 * NHWC, c2 may be 0) -> stats[n][32][2]. workspace: dbir_gn_workspace_floats() floats,
 * zero-initialised once by the caller; its layout is per image, so one workspace sized for the
 * largest batch serves calls of any smaller batch. Replaces the statistics half of GroupNorm32
 * (util.py:191-193, eps 1e-5) / Normalize (attention.py:48-51, vae.py:18-21, eps 1e-6) and
 * the torch.cat before output-block ResBlocks (controlnet.py:39-44).
 * dbir_gn_apply: out = silu?(gn(x)) as op16 NHWC, optionally 2x nearest-upsampled
 * (unet.py:76-78, vae.py:37-40); do_norm = 0 gives a plain cast (operand of Down/Upsample
 * convs, 1x1 skip convs); out_raw (optional) receives the un-normalised cast.
 * dbir_layernorm: op16 out[rows, ldo] = LN(x[rows, c]) (attention.py:257-259,
 * swinir.py:208,214,722,783; eps 1e-5); columns [c, ldo) are zero-filled. c <= 1536 (ldo <= 1280 when c <= 1280).
 */
int64_t dbir_gn_workspace_floats(int32_t n, int32_t hw, int32_t c);
/* Per-(image, group) mean / rstd from the partial sums dbir_gemm emitted while writing the tensor(s)
 * (virtual concat of two tensors: partials1 [n][slots1][c1][2], partials2 [n][slots2][c2][2] or NULL).
 * hw = pixels per image. Deterministic (fixed summation order, fp64 combine). */
int dbir_gn_finalize(const float* partials1, int32_t slots1, int32_t c1, const float* partials2,
                     int32_t slots2, int32_t c2, int32_t n, int32_t hw, float eps, float* stats,
                     void* stream);
int dbir_gn_stats(const float* src1, const float* src2, int32_t c1, int32_t c2, int32_t n,
                  int32_t hw, float eps, float* stats, float* workspace, void* stream);
int dbir_gn_apply(const float* src1, const float* src2, int32_t c1, int32_t c2, int32_t n,
                  int32_t h, int32_t w, const float* stats, const float* gamma,
                  const float* beta, int32_t do_norm, int32_t do_silu, int32_t upsample,
                  void* out, void* out_raw, int32_t imgs_per_group, void* stream);
int dbir_layernorm(const float* x, int64_t ldx, int32_t rows, int32_t c, const float* gamma,
                   const float* beta, float eps, void* out, int64_t ldo, int32_t out_kind,
                   int32_t rows_per_group, void* stream);   /* out_kind 0 = fp32, 1 = op16 */
/* Tiled-VAE GroupNorm (non-fast mode of the reference's utils/tilevae/tilevae.py:177-278): each tile of an
 * image is normalised with the pixel-weighted average of the tiles' own per-group means and biased variances.
 * dbir_gn_moments: fp64 (mean, biased var) per (batch entry, group) -> moments[e][32][2] at e = entry[j]
 *   (device int32 [n]) or entry0 + j when entry is NULL. The source is either the partial sums a conv-mode
 *   dbir_gemm emitted (partials [n][slots][c][2], x NULL) or a fp32 NHWC tensor x [n][hw][c] (partials NULL;
 *   workspace: dbir_gn_moments_workspace_floats() floats, no initialisation needed).
 * dbir_gn_merge: for every image, the weights pixels[e] / sum of its entries' pixels, mean = sum w * mean_e,
 *   var = sum w * var_e (fp64, entries visited in index order, or backwards when reverse = 1) -> (mean, rstd)
 *   of every entry of that image in the stats[e][32][2] layout dbir_gn_apply reads. image: device int32
 *   [entries] in [0, images); pixels: device int64 [entries]. Deterministic. */
int64_t dbir_gn_moments_workspace_floats(int32_t n, int32_t hw, int32_t c);
int dbir_gn_moments(const float* partials, int32_t slots, const float* x, int32_t c, int32_t n, int32_t hw,
                    float* workspace, const int32_t* entry, int32_t entry0, double* moments, void* stream);
int dbir_gn_merge(const double* moments, const int64_t* pixels, const int32_t* image, int32_t entries,
                  int32_t images, int32_t reverse, float eps, float* stats, void* stream);
/* imgs_per_group / rows_per_group > 0: stacked twin problems (see dbir_gemm_args.groups) -- image n /
 * row r takes gamma / beta at offset (n / imgs_per_group) * C resp. (r / rows_per_group) * c. 0 = one set. */

/* ---- SwinIR / SCUNet / Swin-L window attention -------------------------------------------
 * window = 12 (RAM++'s Swin-L encoder, ram/models/swin_transformer.py:68-273): head_dim 32, any head count,
 *   shift 0 or 6, h and w multiples of 12, ldq a multiple of 8 and qkv 16-byte aligned; tensor-core kernel, same
 *   contract as below otherwise. window = 8: */
/* One 8x8 window per CTA; qkv op16 [batch*h*w, ldq] with columns [q | k | v] x (heads, dim)
 * as produced by WindowAttention.qkv (swinir.py:104,122-123); out op16 [batch*h*w, ldo]
 * (first heads*dim columns) in original token order. shift = 0 (W-MSA) or 4 (SW-MSA):
 * replaces torch.roll + window_partition + q k^T + bias + mask + softmax + @v +
 * window_reverse + roll (swinir.py:120-151, 255-276).
 * (heads, head_dim) = 6 x 30 (SwinIR) or {1,2,4,8} x 32 (SCUNet's WMSA, scunet.py:9-99: same roll / window /
 * relative-position-bias / region-mask structure); mask_value is added to the logits of token pairs from
 * different shift regions (-100 in SwinIR, -inf in SCUNet).
 */
int dbir_window_attention(const void* qkv, int64_t ldq, int32_t batch, int32_t h, int32_t w, int32_t heads,
                          int32_t head_dim, int32_t window, int32_t shift, const float* bias_table, float mask_value,
                          void* out, int64_t ldo, void* stream);

/* ---- RAM++ (ram/models/ram_plus.py) --------------------------------------------------------
 * dbir_swin_patch_merge: PatchMerging (swin_transformer.py:294-331) up to its reduction GEMM: x fp32 [n*h*w, ldx]
 *   (first c columns) -> op16 out[n*(h/2)*(w/2), ldo] = LN over 4c (gamma / beta fp32 [4c]) of the concat
 *   [x(2i, 2j) | x(2i+1, 2j) | x(2i, 2j+1) | x(2i+1, 2j+1)].
 * dbir_token_mean: x fp32 [n*tokens, ldx] -> op16 out[n*(tokens+1), ldo]: per image the mean of its tokens
 *   (AdaptiveAvgPool1d, summed in token order) followed by the tokens themselves (swin_transformer.py:571-576).
 * dbir_label_reweight: generate_tag's reweighting (ram_plus.py:291-309): for image b (cls row at cls + b*ld_cls,
 *   dim = 512 floats) and class k, p = softmax_j(scale * cls/|cls| . e[k*per_class + j]) over per_class <= 64
 *   descriptions of label_embed (op16 [classes*per_class, 512]), out row b*classes + k = sum_j p_j e_j (op16).
 */
int dbir_swin_patch_merge(const float* x, int64_t ldx, int32_t n, int32_t h, int32_t w, int32_t c, const float* gamma,
                          const float* beta, float eps, void* out, int64_t ldo, void* stream);
int dbir_token_mean(const float* x, int64_t ldx, int32_t n, int32_t tokens, int32_t c, void* out, int64_t ldo,
                    void* stream);
int dbir_label_reweight(const float* cls, int64_t ld_cls, int32_t batch, const void* label_embed, int32_t classes,
                        int32_t per_class, int32_t dim, float scale, void* out, int64_t ldo, void* stream);

/* ---- face detector / face parser (unaligned-face loop; facexlib RetinaFace-ResNet50 and ParseNet) -----------------
 * dbir_face_input: uint8 HWC pixels [n*h*w, 3] -> op16 [n*h*w, 3], out[c] = (src[c'] * scale - shift_c) / div with
 *   c' = 2 - c when reverse (RetinaFace: minus (104, 117, 123); ParseNet: img2tensor's channel swap, (x/255 - .5)/.5).
 * dbir_patch_gather: patch matrix of a ksize x ksize (1, 3, 7) convolution with stride 1 or 2, pad ksize/2 (zeros, or
 *   reflection when reflect = 1), optionally on the nearest-2x up-sampled input (up2 = 1): op16 x NHWC [n, h, w, ldx]
 *   (first c channels) -> op16 out [n*ho*wo, kpad], column tap*c + ch (taps row-major), columns >= ksize^2 c zero;
 *   kpad a multiple of 64. Feeds dbir_gemm's matrix mode for the convolutions its conv mode does not take.
 * dbir_maxpool3s2: 3x3 / stride 2 / pad 1 max pool, op16 NHWC, c % 8 == 0 (resnet50 stem).
 * dbir_fpn_add_up: op16 out = a + F.interpolate(b, size=(h, w), mode="nearest") with PyTorch's index rule; a fp32
 *   NHWC [n, h, w, c], b op16 NHWC [n, hb, wb, c].
 * dbir_relu_cast: y = relu(x) (fp32, y may be x or NULL) and its op16 copy y16; x = conv + identity (bottleneck tail).
 * dbir_retinaface_decode: head fp32 [rows, 32] (per pixel of the three levels, back to back: class logits 2x2 | box
 *   2x4 | landmarks 2x10) of an h x w input -> out fp32 [2 rows, 15] = x1 y1 x2 y2 score l1x l1y .. l5x l5y per prior
 *   (PriorBox order, min sizes 16/32, 64/128, 256/512, steps 8/16/32, variances 0.1/0.2), in input pixels.
 * dbir_parse_mask: per row of fp32 logits [rows, ld], argmax over `classes` (first maximum) -> uint8 255 for the
 *   face classes of FaceRestoreHelper's colormap (1-13, 15), else 0.
 */
int dbir_face_input(const uint8_t* img, int32_t n, int32_t h, int32_t w, float scale, float shift0, float shift1,
                    float shift2, float div, int32_t reverse, void* out, void* stream);
int dbir_patch_gather(const void* x, int64_t ldx, int32_t n, int32_t h, int32_t w, int32_t c, int32_t ksize,
                      int32_t stride, int32_t reflect, int32_t up2, int32_t kpad, void* out, void* stream);
int dbir_maxpool3s2(const void* x, int32_t n, int32_t h, int32_t w, int32_t c, void* out, void* stream);
int dbir_fpn_add_up(const float* a, const void* b, int32_t n, int32_t h, int32_t w, int32_t hb, int32_t wb, int32_t c,
                    void* out, void* stream);
int dbir_relu_cast(const float* x, int64_t numel, float* y, void* y16, void* stream);
int dbir_retinaface_decode(const float* head, int32_t h, int32_t w, float* out, void* stream);
int dbir_parse_mask(const float* logits, int64_t ld, int64_t rows, int32_t classes, uint8_t* out, void* stream);

/* ---- LLaVA captioner language model (LLaMA-7B, transformers' modeling_llama.py as loaded by the reference's
 * llava/model/language_model/llava_llama.py; decode loop = LlavaLlamaForCausalLM.generate in utils/caption.py:52-145)
 * Every length or position that changes per generated token is a DEVICE int32 scalar, so one captured decode graph
 * replays for every token. KV caches are op16 [capacity, heads, 128].
 * dbir_rmsnorm: LlamaRMSNorm: op16 out[r] = w * x[r] / sqrt(mean(x[r]^2) + eps) over c fp32 columns (per-layer
 *   input_layernorm / post_attention_layernorm and the final norm). c, ldx, ldo multiples of 4.
 * dbir_rope_kv: rows of the fused QKV product (fp32 [rows, ldqkv], columns [q | k | v] x heads x 128) at positions
 *   p0[0] + i: rotary embedding (apply_rotary_pos_emb, rotate_half form, inv_freq = theta^(-2j/128)) of q and k in
 *   fp32; q -> op16 [rows, ldq], k and v -> the caches at row p0[0] + i (LlamaAttention + DynamicCache.update).
 * dbir_attention_causal: prefill: queries q op16 [sq, ldq] at positions 0 .. sq-1 against cache rows 0 .. sq-1,
 *   causal, scale 128^-0.5, tensor cores (mma.sync) -> op16 out [sq, ldo] (LlamaAttention with the causal mask).
 * dbir_attention_decode: one query row per head (q op16 [heads*128]) against cache rows 0 .. len[0]-1
 *   (1 <= len[0] <= capacity), split over 64-key chunks, combined in chunk order (deterministic) -> op16 out
 *   [heads*128]. ws: dbir_attention_decode_ws_bytes(heads, capacity) bytes, no initialisation needed.
 * dbir_gemv: y = W x for one row: W op16 [N, ldw] (K contiguous: the packed weight dbir_gemm reads), x op16 [K],
 *   fp32 accumulation. epilogue 0: y = Wx (QKV, lm_head); 1: y = Wx + residual (fp32 [N]; y may be the residual:
 *   o_proj, down_proj); 2: SwiGLU over rows packed per `pack`-row tile as [values | gates] (dbir_gemm's geglu 2
 *   packing with force_bn = pack): y[c] = values . x * silu(gates . x), N/2 outputs. out_kind 0 fp32, 1 op16.
 * dbir_argmax: first maximum of fp32 logits [n] -> *token (greedy decoding, temperature 0); then each of
 *   advance[0 .. n_advance-1] (device int32) is incremented by one: the decode step's position and length.
 * dbir_embed_gather: fp32 out[i, ldo] = embed_tokens[ids[i]] (op16 [vocab, dim]; ids device int32 [n]).
 * Batched decode (B sequences at the same position, each with its own KV cache; every row's bits equal the
 * single-sequence call on that row):
 * dbir_rope_kv_seqs: row b of qkv is sequence b at position p0[0]; its k / v go to row p0[0] of cache b, which starts
 *   cache_stride elements after cache b - 1.
 * dbir_attention_decode_seqs: query row b (q op16 [B, ldq]) against the first len[0] rows of cache b -> out [B, ldo].
 *   ws: B * dbir_attention_decode_ws_bytes(heads, capacity) bytes.
 * dbir_gemv_rows: dbir_gemv over M <= 8 input rows (x op16 [M, ldx], residual / y [M, ldr] / [M, ldy]): each weight
 *   row is read once for all M inputs; each row's sum runs in the single-row order.
 * dbir_argmax_rows: dbir_argmax of each of M logit rows [M, ld] -> token[0 .. M-1]; advance is incremented once.
 */
int dbir_rmsnorm(const float* x, int64_t ldx, int32_t rows, int32_t c, const float* w, float eps, void* out, int64_t ldo,
                 void* stream);
int dbir_rope_kv(const float* qkv, int64_t ldqkv, int32_t rows, int32_t heads, const int32_t* p0, float theta, void* q,
                 int64_t ldq, void* k_cache, void* v_cache, void* stream);
int dbir_attention_causal(const void* q, int64_t ldq, const void* k_cache, const void* v_cache, int32_t heads, int32_t sq,
                          void* out, int64_t ldo, void* stream);
int64_t dbir_attention_decode_ws_bytes(int32_t heads, int32_t capacity);
int dbir_attention_decode(const void* q, const void* k_cache, const void* v_cache, int32_t heads, int32_t capacity,
                          const int32_t* len, void* ws, int64_t ws_bytes, void* out, void* stream);
int dbir_gemv(const void* w, int64_t ldw, const void* x, int32_t N, int32_t K, int32_t epilogue, int32_t pack,
              const float* residual, void* y, int32_t out_kind, void* stream);
int dbir_argmax(const float* logits, int32_t n, int32_t* token, int32_t* advance, int32_t n_advance, void* stream);
int dbir_embed_gather(const void* table, int32_t vocab, const int32_t* ids, int32_t n, int32_t dim, float* out,
                      int64_t ldo, void* stream);
int dbir_rope_kv_seqs(const float* qkv, int64_t ldqkv, int32_t seqs, int32_t heads, const int32_t* p0, float theta,
                      void* q, int64_t ldq, void* k_cache, void* v_cache, int64_t cache_stride, void* stream);
int dbir_attention_decode_seqs(const void* q, int64_t ldq, const void* k_cache, const void* v_cache,
                               int64_t cache_stride, int32_t seqs, int32_t heads, int32_t capacity, const int32_t* len,
                               void* ws, int64_t ws_bytes, void* out, int64_t ldo, void* stream);
int dbir_gemv_rows(const void* w, int64_t ldw, const void* x, int64_t ldx, int32_t M, int32_t N, int32_t K,
                   int32_t epilogue, int32_t pack, const float* residual, int64_t ldr, void* y, int64_t ldy,
                   int32_t out_kind, void* stream);
int dbir_argmax_rows(const float* logits, int64_t ld, int32_t M, int32_t n, int32_t* token, int32_t* advance,
                     int32_t n_advance, void* stream);

/* ---- small / memory-bound ops ------------------------------------------------------------
 * conv3x3_small_cin : stems with <= 16 input channels; input = virtual concat of two NCHW
 *   fp32 tensors scaled by in_scale/in_shift; weight fp32 [9*Cin, Cout]; out NHWC fp32
 *   (unet.py:500-506, controlnet.py:158-166,316; vae.py:322-324,482-484).
 * conv3x3_small_cout: heads with 3/4/8 output channels; op16 NHWC in, weight fp32
 *   [Cout, 9*Cin], out = (conv + bias) * post_scale + post_shift[c], NCHW or NHWC fp32
 *   (unet.py:675-679 out conv; vae.py:340-345,520-522; swinir.py:811,885-887).
 * im2col_s2: 3x3 stride-2 patches of fp32 NHWC -> op16 [n*ho*wo, 9c] for dbir_gemm
 *   (Downsample unet.py:99 pad_lo=1; vae.py:51-55 pad_lo=0).
 * linear_f32: y = act_out(act_in(x) W^T + b), small row counts, all fp32
 *   (time_embed / emb_layers unet.py:166-172,494-498,616-617; quant convs vae.py:569-570).
 * timestep_embedding: util.py:128-148. softmax_rows: vae.py:232-282 (mid attention).
 * sampler_step: CFG mix + x0 + posterior / DDIM update, one launch per step
 *   (spaced_sampler.py:118-184, ddim_sampler.py:98-146); coef -> 8 floats of the step.
 * tile_gather / tile_blend: mixture-of-diffusers tiling (utils/common.py:123-232).
 */
int dbir_conv3x3_small_cin(const float* in1, const float* in2, int32_t c1, int32_t c2, int32_t n,
                           int32_t h, int32_t w, const float* weight_kc, const float* bias,
                           int32_t cout, float in_scale, float in_shift, float* out_nhwc,
                           void* stream);
int dbir_conv3x3_small_cout(const void* in_nhwc, int32_t n, int32_t h, int32_t w, int32_t cin,
                            const float* weight, const float* bias, int32_t cout,
                            float post_scale, const float* post_shift, float* out,
                            int32_t out_nchw, void* stream);
int dbir_im2col_s2(const float* in_nhwc, int32_t n, int32_t h, int32_t w, int32_t c,
                   int32_t pad_lo, void* out, void* stream);
int dbir_linear_f32(const float* x, int64_t ldx, int32_t m, int32_t k, const float* weight,
                    const float* bias, int32_t n, int32_t silu_in, int32_t silu_out, float* y,
                    int64_t ldy, void* stream);
int dbir_timestep_embedding(const float* t, int32_t m, int32_t dim, float* out, void* stream);
/* y = alpha * x + z over fp32 rows [rows, c] (z may be NULL); writes fp32 y (may be NULL) and/or an op16 copy
 * with row stride ld16 -- the tails of RRDBNet's dense blocks, `out * 0.2 + x` (bsrnet.py:69-70,85-87), and the
 * operand cast of a block output into the next block's concat buffer. */
int dbir_axpby_cast(const float* x, float alpha, const float* z, int64_t rows, int32_t c, float* y, void* y16,
                    int64_t ld16, void* stream);
int dbir_softmax_rows(const float* s, int64_t lds, int32_t rows, int32_t cols, float scale,
                      void* out, int64_t ldo, void* stream);
int dbir_upsample2x_op16(const void* in, int32_t n, int32_t h, int32_t w, int32_t c, void* out,
                         void* stream);
int dbir_swin_stem(const float* in_nchw, int32_t n, int32_t h, int32_t w, int32_t r,
                   const float* mean3, float range, int32_t cpad, void* out, void* stream);
int dbir_nchw_to_nhwc(const float* in, int32_t n, int32_t c, int32_t hw, float* out, void* stream);
int dbir_nhwc_to_nchw(const float* in, int32_t n, int32_t c, int32_t hw, float* out, void* stream);
int dbir_sampler_step(const float* eps_cond, const float* eps_uncond, float cfg_scale,
                      const float* x, const float* noise, const float* coef, int32_t mode,
                      int64_t numel, float* x_out, void* stream);
int dbir_tile_gather(const float* full, int32_t b, int32_t c, int32_t h, int32_t w,
                     const int32_t* coords, int32_t ntiles, int32_t tile, float* tiles,
                     void* stream);
int dbir_tile_blend(const float* tiles, int32_t b, int32_t c, int32_t h, int32_t w,
                    const int32_t* coords, int32_t ntiles, int32_t tile, const float* weights,
                    float* out, void* stream);

/* ---- fused output epilogue -------------------------------------------------------------
 * fixed = high_freq((sample + 1) / 2) + low_freq(style): wavelet_reconstruction (utils/common.py:29-77,
 * 5-level a-trous decomposition, replicate padding) of the decoded sample (NCHW view, [-1, 1]) against
 * the stage-1 image (NCHW view, [0, 1]); element strides per image / channel / row, unit column stride.
 * out_u8 != NULL: uint8 NHWC trunc(clamp(fixed * 255, 0, 255)) -- the tail of Pipeline.run
 * (pipeline.py:306-320) when no resize follows; else out_f32 receives `fixed` as contiguous NCHW fp32.
 */
int dbir_wavelet_fix(const float* sample, int64_t s_img, int64_t s_ch, int64_t s_row,
                     const float* style, int64_t t_img, int64_t t_ch, int64_t t_row,
                     int32_t batch, int32_t h, int32_t w, void* out_u8, float* out_f32, void* stream);

/* ---- Real-ESRGAN degradation (dataset/batch_transform.py:142-285) -----------------------------
 * fp32 NCHW in and out, contiguous. The random draws stay with the caller (torch generators); these
 * entries compute what lies between them. Per-sample parameters are passed as the raw uniform draws u
 * with param = u * span + lo and gray = (u_gray < gray_prob), evaluated on the device.
 * filter2d: utils.py:162-187, reflect padding, odd k <= 63, h and w > k/2. kernel [kb, k, k] with
 *   kernel_stride = k*k (one per sample) or 0 (one for the batch). sub != NULL filters the USM threshold
 *   mask (|x - sub| * 255 > threshold) instead of x (utils.py:205-207).
 * resize: F.interpolate, align_corners=False, no antialias; mode 0 area (adaptive_avg_pool2d bins),
 *   1 bilinear, 2 bicubic (A = -0.75). ratio = source/destination coordinate scale: 1/scale_factor
 *   for the scale_factor= form, in/out for the size= form.
 * gaussian_noise: degradation.py:461-554; noise [b,c,h,w] and noise_gray [h,w] (or NULL) are torch.randn draws.
 * noise_levels: q = clamp(round(x*255), 0, 255)/255 (gray = 1: of rgb_to_grayscale(x), one channel) and the
 *   256-bin level histogram per sample, hist int32 [b, 256] (zeroed here).
 * poisson_rate: vals[s] = 2^ceil(log2(distinct levels of sample s)), rate = q * vals (torch.poisson's input).
 * poisson_noise: degradation.py:610-724: noise = draw/vals - q, mixed with the gray field's when q_gray != NULL,
 *   times the scale; out = clip(img + noise, 0, 1).
 * diffjpeg: diffjpeg.py:450-492 with differentiable=False; quality [b]: with quality_is_factor = 0 the quality of
 *   each sample, turned into its table factor on the device as PyTorch does for a tensor quality; with 1 the factors
 *   themselves (a Python-number quality, whose factor the reference computes in double on the host).
 *   clamp_in = 1 clamps the input to [0, 1] first (batch_transform.py:192,255,260).
 * usm_blend: utils.py:208-210, soft = filter2d of the threshold mask.
 * lq_levels: clamp(round(x*255), 0, 255)/255 (batch_transform.py:271).
 * pair_nhwc: lq -> NHWC, hq*2-1 -> NHWC (batch_transform.py:279-281).
 */
int dbir_filter2d(const float* x, const float* sub, float threshold, int32_t b, int32_t c, int32_t h, int32_t w,
                  const float* kernel, int64_t kernel_stride, int32_t k, float* out, void* stream);
int dbir_resize(const float* x, int64_t planes, int32_t hin, int32_t win, int32_t hout, int32_t wout, int32_t mode,
                float ratio_h, float ratio_w, float* out, void* stream);
int dbir_gaussian_noise(const float* img, const float* noise, const float* noise_gray, const float* u_sigma,
                        float sigma_lo, float sigma_span, const float* u_gray, float gray_prob, int32_t b, int32_t c,
                        int64_t hw, float* out, void* stream);
int dbir_noise_levels(const float* img, int32_t b, int32_t c, int64_t hw, int32_t gray, float* q, int32_t* hist,
                      void* stream);
int dbir_poisson_rate(const float* q, const int32_t* hist, int32_t b, int64_t per_sample, float* vals, float* rate,
                      void* stream);
int dbir_poisson_noise(const float* img, const float* q, const float* draw, const float* vals, const float* q_gray,
                       const float* draw_gray, const float* vals_gray, const float* u_scale, float scale_lo,
                       float scale_span, const float* u_gray, float gray_prob, int32_t b, int32_t c, int64_t hw,
                       float* out, void* stream);
int dbir_diffjpeg(const float* x, const float* quality, int32_t quality_is_factor, int32_t b, int32_t h, int32_t w,
                  int32_t clamp_in, float* out, void* stream);
int dbir_usm_blend(const float* img, const float* blur, const float* soft, float weight, int64_t n, float* out,
                   void* stream);
int dbir_lq_levels(const float* x, int64_t n, float* out, void* stream);
int dbir_pair_nhwc(const float* lq, const float* hq, int32_t b, int32_t c, int64_t hw, float* lq_out, float* hq_out,
                   void* stream);

/* ---- Brownian tree (noise of the dpm++_sde step rule, sampler/k_diffusion.py:70-120, 548-586) ----------------
 * brownian_increment: out[e] = W_e(t1) - W_e(t0) (fp32) for e < n, where W_e is a Brownian motion on [lo, hi] with
 *   W_e(lo) = 0, the same for every call with the same (seed, lo, hi, depth). W(t) walks `depth` levels of the dyadic
 *   bisection of [lo, hi]: each midpoint is a Brownian-bridge draw between its interval's end values, and below the
 *   last level W(t) is one more bridge draw between the leaf's ends, keyed with t. t0 and t1 are clamped to [lo, hi].
 *   Every draw is a Philox4x32-10 normal (Box-Muller) keyed by (seed, node, element); the walk runs in fp64.
 *   0 <= depth <= 62; pick it so that (hi - lo) / 2^depth is the tolerance wanted.
 * brownian_increment_samples: one tree per sample of a batch: out[b * n + e] (b < samples, e < n) is element e of
 *   brownian_increment with seed seeds[b] (seeds: device uint64 [samples]), bit for bit.
 * brownian_draws: the raw draws that walk uses, for checking the stream: for e < n, the four Philox words
 *   (words_out uint32 [n, 4]) and the normal (normals fp64 [n]) of element e at `node` (heap numbering: 0 is W(hi),
 *   1 the midpoint of [lo, hi], 2k and 2k + 1 the midpoints of node k's halves), or with leaf = 1 of the leaf draw
 *   at time t. Either output may be NULL.
 */
int dbir_brownian_increment(float* out, int64_t n, uint64_t seed, double lo, double hi, double t0, double t1,
                            int32_t depth, void* stream);
int dbir_brownian_increment_samples(float* out, int64_t n, int32_t samples, const uint64_t* seeds, double lo,
                                    double hi, double t0, double t1, int32_t depth, void* stream);
int dbir_brownian_draws(uint32_t* words_out, double* normals, int64_t n, uint64_t seed, uint64_t node, int32_t leaf,
                        double t, void* stream);

/* ---- face paste-back (utils/face.py FaceRestoreHelper.paste_faces_to_input_image) ---------------------------
 * Byte-identical restatement of the cv2 / numpy paste of the unaligned-face loop, one face at a time over a region of
 * interest (x0, y0, rw, rh) of the h x w frame: a rectangle that holds every pixel where the face's warped square,
 * soft mask or warped parse mask can be non-zero. ROI buffers are fp32 [rh, rw]; borders are the frame's.
 * `map` is a HOST pointer to the 6 doubles of the destination -> source map (cv2.warpAffine's inverted matrix).
 * paste_square: cv2.erode(cv2.warpAffine(ones(fs, fs) f32, inv, (w, h)), 2x2 ones) over the ROI; *sum (device fp64)
 *   receives the ROI's sum.
 * paste_soft: cv2.GaussianBlur(cv2.erode(square, (2e)x(2e) ones), (2e+1, 2e+1), 0) over the ROI, taps (device f32
 *   [2e+1]) = cv2.getGaussianKernel(2e+1, 0, CV_32F). edge 0 or >= 3, w a multiple of 4 (cv2's per-column tap
 *   order is restated for those). tmp: ROI-sized scratch.
 * paste_parse_blur: masks u8 [n, size, size] -> out f64: two cv2.GaussianBlur((k, k)) with taps (device f64 [k]),
 *   the 10-pixel frame zeroed, / 255. tmp: same size as out.
 * paste_compose: for every sample s < samples, out[s] (f64 [h, w, 3]) = mask * pasted + (1 - mask) * out[s] over the
 *   ROI, with inv_restored = warpAffine(faces[s] u8 [fs, fs, 3]), pm = warpAffine(pms[s] f64 [fs, fs]),
 *   pasted = square * inv_restored (f32) and mask = min(pm, soft). faces / pms advance by face_stride / pm_stride
 *   elements per sample.
 * paste_begin: out f64 = img u8 (n elements); paste_end: img = astype(uint8) (truncation) of in.
 */
int dbir_paste_square(const double* map, int32_t face_size, int32_t h, int32_t w, int32_t x0, int32_t y0, int32_t rw,
                      int32_t rh, float* square, double* sum, void* stream);
int dbir_paste_soft(const float* square, int32_t h, int32_t w, int32_t x0, int32_t y0, int32_t rw, int32_t rh,
                    int32_t edge, const float* taps, float* tmp, float* soft, void* stream);
int dbir_paste_parse_blur(const uint8_t* masks, int32_t n, int32_t size, const double* taps, int32_t k, double* tmp,
                          double* out, void* stream);
int dbir_paste_compose(const uint8_t* faces, int64_t face_stride, const double* pms, int64_t pm_stride,
                       int32_t samples, const float* square, const float* soft, const double* map, int32_t face_size,
                       int32_t h, int32_t w, int32_t x0, int32_t y0, int32_t rw, int32_t rh, double* out,
                       void* stream);
int dbir_paste_begin(const uint8_t* img, int64_t n, double* out, void* stream);
int dbir_paste_end(const double* in, int64_t n, uint8_t* img, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* DIFFBIR_B200_H */
