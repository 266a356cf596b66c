/*
 * visrag_b200 — C ABI of the H100-native (sm_90a) VisRAG-Ret embedding + retrieval hot path.
 *
 * The reference (OpenBMB/VisRAG) is pure Python: it has no FFI for this path. The
 * drop-in boundary is the three Python call signatures of SURVEY.md §8(b); this C ABI
 * is what sits underneath the Python mirror of those signatures
 * (visrag_b200/{modeling,encoder,retriever}.py), and each entry point below names the
 * reference code whose GPU work it replaces (paths relative to the reference repo).
 *
 * Conventions
 *  - every pointer is a DEVICE pointer unless the name ends in _host; the caller owns
 *    all buffers (inputs, outputs, workspaces); the library allocates nothing;
 *  - all work is enqueued on the caller's cudaStream_t (passed as void*); no hidden
 *    synchronisation, so every call is CUDA-graph capturable;
 *  - return value: 0 on success, non-zero on error; vr_last_error() returns a
 *    thread-local message; nothing throws or exits across the ABI;
 *  - row-major matrices; "ld*" = leading dimension in ELEMENTS;
 *  - "Alignment (bytes) of <entry point>: <pointer> <n>, ..." lines give the base alignment each pointer needs: the
 *    widest vector access the kernels make to it (with the ld / dim rules of each call, every row is then aligned too).
 *    A pointer below its alignment is refused (return 2, the message names it) before any CUDA call; NULL optional
 *    pointers are exempt.
 */
#ifndef VISRAG_B200_H
#define VISRAG_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VR_ABI_VERSION 2

typedef enum { VR_BF16 = 0, VR_F16 = 1, VR_F32 = 2 } vr_dtype;

const char* vr_last_error(void);
int vr_abi_version(void);

/* ------------------------------------------------------------------------------------
 * Dense contraction  C[M,N] = A[M,K] * B[N,K]^T  on wgmma tensor cores (TMA-staged
 * 128B-swizzled tiles -> warpgroup MMA -> fp32 accumulators in registers -> fused epilogue).
 * Replaces every nn.Linear / Conv2d-as-GEMM the reference dispatches to cuBLAS/cuDNN:
 *   timm/layers/patch_embed.py:87 (patch conv), timm/models/vision_transformer.py:88,105
 *   (qkv, proj), timm/layers/mlp.py:41-49 (fc1+GELU, fc2), resampler.py:154,159-167,
 *   modeling_minicpm.py:850-852,908 (q,k,v,o), modeling_minicpm.py:333 (SwiGLU MLP).
 * A and B are both bf16 (ab_dtype = VR_BF16) or both fp16 (VR_F16); K*2 bytes and lda/ldb*2 bytes must be
 * multiples of 16 (TMA); N must be a multiple of 8. Every block_n selector runs both operand types; the accumulator,
 * bias, residual, row add and RoPE tables are fp32 either way. Output types:
 *   bf16 operands: LINEAR writes VR_BF16 or VR_F32 (out_dtype); ROPE / SWIGLU write bf16 (out_dtype is not read);
 *   fp16 operands: LINEAR writes VR_F16 or VR_F32; ROPE / SWIGLU write fp16 and need out_dtype = VR_F16;
 *   GELU writes the operands' 16-bit type only. Any other combination is refused before any CUDA call.
 * An fp16 output rounds to nearest with no clamp: a value beyond 65504 is stored as inf.
 * A LINEAR out must be 16-byte aligned (refused before any CUDA call otherwise); with ldo % 8 == 0 every row then is.
 * Alignment (bytes) of vr_gemm: A 16, B 16, bias 8, rowadd 8, resid 8, rope_cos 8, rope_sin 8, positions 4, out 16 (LINEAR), out 4 (ROPE, SWIGLU)
 * ---------------------------------------------------------------------------------- */
typedef enum {
    VR_EPI_LINEAR = 0, /* out = [resid +] scale*(gelu?(acc + bias)) [+ rowadd[row % period]] */
    VR_EPI_ROPE = 1,   /* MiniCPM q|k|v: rotate-half RoPE on 64-wide heads in columns < rope_cols; 16-bit out */
    VR_EPI_SWIGLU = 2  /* B rows interleaved [32 gate | 32 up] per 64: out[:, j] = silu(g_j)*u_j; 16-bit, N/2 cols */
} vr_epi_mode;

typedef struct {
    int32_t mode;          /* vr_epi_mode */
    int32_t out_dtype;     /* LINEAR: VR_F32 or the operands' type; ROPE / SWIGLU: VR_F16 with fp16 operands, else unread */
    int32_t act_gelu;      /* LINEAR: exact erf-GELU applied to (acc + bias) */
    float scale;           /* LINEAR: multiplies the activation before the residual add */
    const float* bias;     /* [N] fp32 or NULL */
    const float* resid;    /* [M, ldo] fp32 or NULL; may alias out (in-place residual stream) */
    const float* rowadd;   /* [period, N] fp32 or NULL (ViT position embedding) */
    int32_t rowadd_period; /* rows of rowadd; row index used is (row % period) */
    const int32_t* positions; /* ROPE: [M] position of each packed token inside its sequence */
    const float* rope_cos; /* ROPE: [max_pos, 32] fp32 */
    const float* rope_sin; /* ROPE: [max_pos, 32] fp32 */
    int32_t rope_cols;     /* ROPE: columns [0, rope_cols) are rotated (q and k); the rest (v) pass through */
    void* out;             /* [M, ldo] */
    int64_t ldo;
} vr_gemm_epilogue;

int vr_gemm(const void* A, int64_t lda, const void* B, int64_t ldb, int32_t ab_dtype, int32_t M, int32_t N, int32_t K,
            const vr_gemm_epilogue* epi, void* stream);

/* Same operation with the tile shape chosen by the caller (benchmarks, parity tests of every variant):
 *   block_n = 0    what vr_gemm picks: 128 x 64 tiles when M <= 128 (weight-streaming bound: more, narrower tiles), else
 *                  the ping-pong kernel in CTA pairs (block_n = 4)
 *   block_n = 2    ping-pong kernel: 128 x 128 tiles, each owned by one of two consumer warpgroups that take turns on the
 *                  tensor cores, so one tile's epilogue runs under the next tile's MMAs; N tiles ordered in slices whose
 *                  weight fits in L2
 *   block_n = 4    the same in 2-CTA clusters: a pair takes two adjacent M tiles of one N tile and each CTA loads half of
 *                  the B tile, multicast to both
 *   block_n = 5    block_n = 2 with plain n-fastest tile order (measures what the L2 slices buy)
 *   block_n = 256 / 192 / 128 / 64   cooperative kernel, token-major accumulator, 128 tokens x block_n features per tile
 *                  (both consumer warpgroups share a tile and run its epilogue together)
 *   block_n = 3    feature-major accumulator (the weight tile is the MMA's M operand, 128 tokens are its N), LINEAR
 *                  epilogues only */
int vr_gemm_tuned(const void* A, int64_t lda, const void* B, int64_t ldb, int32_t ab_dtype, int32_t M, int32_t N,
                  int32_t K, const vr_gemm_epilogue* epi, int32_t block_n, void* stream);


/* ------------------------------------------------------------------------------------
 * Device image front-end (SURVEY.md 8f.2): Pillow-bit-compatible 8-bit bicubic resampling + grid crop.
 * Replaces the host-side `image.resize(size, Image.BICUBIC)` calls of slice_image
 * (modeling_minicpmv/modeling_minicpmv.py:509,519,531) and split_to_patches (:571-592); the arithmetic is
 * Pillow's ImagingResample (src/libImaging/Resample.c): horizontal pass over source rows
 * [row_first, row_first+row_count) into an 8-bit intermediate, then the vertical pass, 22-bit fixed-point
 * coefficients, 32-bit sums, clip8. Results are bit-identical to PIL.
 *   src        [n, in_h, in_w, src_pixel_bytes] uint8 (n pages of one size); src_pixel_bytes = 3 (packed RGB) or
 *              4 (RGBX: Pillow's native row layout for mode "RGB", so a page can travel without any repacking on
 *              the host; the 4th byte is ignored)
 *   bounds_*   [out, 2] int32 (first source index, tap count); coefficients int32 fixed point as Pillow's
 *              precompute_coeffs + normalize_coeffs_8bpc produce them (frontend.resample_coeffs): coeffs_v
 *              [out_h, ksize_v] (row per output row), coeffs_h TAP-MAJOR [ksize_h, out_w] (coalesced across the
 *              threads of the horizontal pass); NULL for an axis whose size does not change (Pillow skips that
 *              pass). in_w <= 12288.
 *   tmp        workspace of n * row_count * ((out_w*3 + 3) & ~3) bytes (4-byte row pitch), needed when both passes run
 *   out        slice buffer [*, cell_h, cell_w, 3] uint8: the out_h x out_w result of page i is cut into
 *              (out_h/cell_h) x (out_w/cell_w) cells, row-major, stored as slices first_cell[i], first_cell[i]+1, ...
 *              (cell = whole image for the thumbnail). first_cell: [n] int32, device.
 * ---------------------------------------------------------------------------------- */
int vr_resample_u8(const uint8_t* src, int32_t src_pixel_bytes, int32_t n, int32_t in_h, int32_t in_w, const int32_t* bounds_h,
                   const int32_t* coeffs_h, int32_t ksize_h, const int32_t* bounds_v, const int32_t* coeffs_v,
                   int32_t ksize_v, int32_t row_first, int32_t row_count, int32_t out_h, int32_t out_w, uint8_t* tmp,
                   uint8_t* out, const int32_t* first_cell, int32_t cell_h, int32_t cell_w, void* stream);

/* ------------------------------------------------------------------------------------
 * Fused softmax(Q K^T * scale) V on wgmma. S, P (bf16, register A operand of the second MMA), running max / sum and the
 * O accumulator all live in registers. Sequences longer than 64 queries: two consumer warpgroups (128 queries) per CTA
 * share one K/V stream; up to 64 queries per sequence: one warpgroup per CTA. Both forms (and vr_attention_force_v1)
 * give a sequence the same output bits: it does not depend on max_q, on the other sequences of the batch or on the form.
 * Non-finite values: a NaN or inf in one sequence's Q, K or V never reaches another sequence's output. (A sequence's last
 * 128-key tile is read from the packed rows and may hold the next sequence's rows; their scores are masked to -inf and
 * their V rows are zeroed in shared memory before P V, so no p = 0 multiplies a foreign inf or NaN.) Within one causal
 * sequence, a non-finite V at key j can reach earlier rows that share j's 128-key tile (their p_j = 0 times inf is NaN),
 * as a masked softmax followed by a matmul gives; rows whose key tiles all end before j are unaffected.
 * Replaces F.scaled_dot_product_attention in timm/models/vision_transformer.py:92-96 (ViT,
 * 16 heads x 72, no mask), modeling_minicpm.py:895-903 (MiniCPM, causal + right padding ->
 * here: packed var-len sequences, no padding rows at all) and nn.MultiheadAttention in
 * resampler.py:159-163 (64 learned queries x N keys, 18 heads x 128).
 * q/k/v are bf16 (or, with VR_ATTN_F16, fp16) row-major token matrices; head h starts at column *_col0 + h*head_stride
 * (head_stride = head_dim rounded up to a multiple of 16; pad columns must hold zeros).
 * Alignment (bytes) of vr_attention: q 16, k 16, v 16, cu_q 4, cu_k 4, out 4
 * Causal with fewer query rows than key rows (len_q < len_k, e.g. a sequence whose first len_k - len_q rows come from a
 * prefix cache): the query rows are the LAST len_q rows of the sequence. Query i of sequence b attends keys
 * j <= i + (len_k - len_q), and its output row has the same bits as row len_k - len_q + i of the full causal run over the
 * same keys: key tiles start at the same 128-key offsets from the sequence start, and a tile that lies wholly past a
 * row's last key adds nothing to that row.
 * ---------------------------------------------------------------------------------- */
typedef struct {
    const void* q;  int64_t ldq;  int64_t q_rows;   /* q_rows: rows in the q buffer (TMA bound) */
    const void* k;  int64_t ldk;
    const void* v;  int64_t ldv;  int64_t kv_rows;  /* rows in the k and v buffers */
    int32_t q_col0, k_col0, v_col0;
    int32_t head_stride;      /* 64, 80 or 128 */
    int32_t head_dim;         /* 64, 72 or 128: output columns per head */
    int32_t heads, batch;
    const int32_t* cu_q;      /* [batch+1] packed query offsets, or NULL: every item uses q rows [0, max_q) */
    const int32_t* cu_k;      /* [batch+1] packed key offsets */
    int32_t max_q, max_k;     /* longest query / key sequence (grid sizing) */
    int32_t causal;
    float scale;
    void* out; int64_t ldo;   /* bf16 (fp16 with VR_ATTN_F16); row = cu_q ? cu_q[b]+i : b*max_q+i ; head h at column h*head_dim */
    int32_t flags;            /* VR_ATTN_* */
} vr_attn_params;

/* The caller guarantees V[:, head_dim] == 1 for every head (head_dim == head_stride - 8; e.g. a bias of 1 in the zero
 * padding of the QKV projection). A kernel may then take the softmax denominator out of the P.V MMA (column head_dim of
 * the accumulator) instead of summing P in registers; the sm_90a kernels sum P in registers (it is already there) and
 * ignore the column. Results are the same up to fp32 summation order. */
#define VR_ATTN_V_ONES_COLUMN 1
/* q, k, v and out are fp16 instead of bf16. P (the softmax numerators, <= 1) is rounded to fp16 for the P.V MMA with
 * round-to-nearest and no flush: p below 2^-14 become fp16 subnormals, not zeros. S, the running max / sum, alpha and the
 * O accumulator stay fp32 and run the same arithmetic as the bf16 form, so the batch-invariance statement above holds for
 * fp16 too (the same bits from either form and any batch). */
#define VR_ATTN_F16 2

int vr_attention(const vr_attn_params* p, void* stream);
/* test / benchmark hook (process-wide): 0 = default dispatch, 1 = always the one-warpgroup (64 queries per CTA) kernel */
void vr_attention_force_v1(int32_t variant);


/* ------------------------------------------------------------------------------------
 * HBM-bound standalone kernels (128-bit vectorised, one pass over the activation).
 * ---------------------------------------------------------------------------------- */

/* uint8 HWC slices -> normalised bf16 patch matrix (ToTensor + Normalize(0.5,0.5) + the unfold of the
 * 14x14/stride-14 patch conv): modeling_minicpmv.py:84-92 + timm/layers/patch_embed.py:87.
 * pixels: [n_slices, h, w, 3] uint8 (h, w multiples of `patch`); out: [n_slices*(h/patch)*(w/patch), ldo] bf16,
 * column c*patch*patch + ky*patch + kx (the Conv2d weight's flattening); columns [3*patch^2, ldo) are zeroed.
 * bf16(fma(u, 2/255, -1)) - bit-identical to bf16((u/255 - 0.5)/0.5) for all 256 byte values. patch <= 85, any w: a strip of
 * `patch` pixel rows that does not fit 200 KB of shared memory (patch 14, ldo 640: w of 4858 and more) is converted in chunks of
 * patch columns, with the same bits. Returns 2 if ldo is so large that its offset table leaves no room for one patch.
 * Alignment (bytes) of vr_im2col_norm: out 16 */
int vr_im2col_norm(const uint8_t* pixels, int32_t n_slices, int32_t h, int32_t w, int32_t patch, void* out, int64_t ldo,
                   void* stream);
/* The same with the output type chosen: out_dtype = VR_BF16 (what vr_im2col_norm writes) or VR_F16, where
 * fp16(fma(u, 2/255, -1)) is likewise bit-identical to fp16((u/255 - 0.5)/0.5) for all 256 byte values. */
int vr_im2col_norm_ex(const uint8_t* pixels, int32_t n_slices, int32_t h, int32_t w, int32_t patch, void* out, int64_t ldo,
                      int32_t out_dtype, void* stream);

/* LayerNorm over the last dim (timm vision_transformer.py:142,155,525; resampler.py:155,166): fp32 in -> bf16 out.
 * If out2 != NULL also writes out2 = LN(x) + add[row % add_period] (bf16) — the resampler's K input (kv + pos).
 * Alignment (bytes) of vr_layernorm: x 16, gamma 16, beta 16, add 16, out 8, out2 8 */
int vr_layernorm(const float* x, int64_t ldx, const float* gamma, const float* beta, float eps, int32_t rows, int32_t dim,
                 void* out, int64_t ldo, void* out2, const float* add, int32_t add_period, void* stream);
/* vr_layernorm with out and out2 written as out_dtype = VR_BF16 (vr_layernorm) or VR_F16; mean, variance and the add of
 * out2 stay fp32, and only the stores round. */
int vr_layernorm_ex(const float* x, int64_t ldx, const float* gamma, const float* beta, float eps, int32_t rows, int32_t dim,
                    void* out, int64_t ldo, void* out2, const float* add, int32_t add_period, int32_t out_dtype, void* stream);

/* RMSNorm (modeling_minicpm.py:119-123): fp32 in -> bf16 out.
 * Alignment (bytes) of vr_rmsnorm: x 16, gamma 16, out 8 */
int vr_rmsnorm(const float* x, int64_t ldx, const float* gamma, float eps, int32_t rows, int32_t dim, void* out, int64_t ldo,
               void* stream);
/* vr_rmsnorm with out written as out_dtype = VR_BF16 (vr_rmsnorm) or VR_F16; statistics in fp32. */
int vr_rmsnorm_ex(const float* x, int64_t ldx, const float* gamma, float eps, int32_t rows, int32_t dim, void* out, int64_t ldo,
                  int32_t out_dtype, void* stream);

/* LM input assembly (modeling_minicpmv.py:139-166): for packed token t,
 *   src[t] >= 0 : h[t] = vision[src[t]]            (resampler output row, fp32)
 *   src[t] <  0 : h[t] = embed[-(src[t]+1)] * scale_emb   (bf16 table)
 * h: [tokens, dim] fp32.
 * Alignment (bytes) of vr_build_lm_input: src 4, embed 8, vision 16, h 16 */
int vr_build_lm_input(const int32_t* src, int32_t tokens, int32_t dim, const void* embed_bf16, float scale_emb,
                      const float* vision, int64_t ldv, float* h, int64_t ldh, void* stream);
/* vr_build_lm_input with the embedding table's type given: embed_dtype = VR_BF16 (vr_build_lm_input) or VR_F16. Either is
 * widened to fp32 exactly and multiplied by scale_emb in fp32; h is fp32. */
int vr_build_lm_input_ex(const int32_t* src, int32_t tokens, int32_t dim, const void* embed, int32_t embed_dtype,
                         float scale_emb, const float* vision, int64_t ldv, float* h, int64_t ldh, void* stream);

/* Final RMSNorm + pooling + L2 normalise (modeling_minicpm.py:1280; dense_retrieval_model.py:170-223):
 * per packed sequence b (rows cu[b]..cu[b+1]) of h [tokens, dim] fp32 -> reps [batch, dim] fp32.
 * pooling: 0 wmean (w_t = t+1), 1 mean, 2 lasttoken, 3 cls. normalise: x / max(||x||, 1e-12).
 * One thread-block cluster of 8 (or 4) CTAs per sequence, every row read once; h, gamma and reps 16-byte aligned; any
 * sequence length (no per-length shared memory), dim <= 4096. A sequence's sums run in one fixed order whatever the
 * cluster size, so its output bits do not depend on the batch size or on the other sequences of the batch.
 * Alignment (bytes) of vr_pool_norm: h 16, gamma 16, cu 4, reps 16 */
int vr_pool_norm(const float* h, int64_t ldh, const float* gamma, float eps, const int32_t* cu, int32_t batch, int32_t dim,
                 int32_t pooling, int32_t normalize, float* reps, void* stream);

/* Prefix-cache row assembly: every sequence b of out becomes [prefix rows ; its own rows]:
 *   out rows [cu_out[b], cu_out[b] + prefix_len)   = prefix rows 0 .. prefix_len - 1
 *   out rows [cu_out[b] + prefix_len, cu_out[b+1]) = rows [cu_rows[b], cu_rows[b+1]) of `rows`
 * so cu_out[b+1] - cu_out[b] = prefix_len + cu_rows[b+1] - cu_rows[b], and out_rows = cu_out[batch]. Each row copies
 * `cols` elements of elem_size bytes (2: the 16-bit K|V block of a qkv row; 4: the fp32 residual stream) from column 0
 * of the given pointers; prefix, rows and out must be 16-byte aligned and cols * elem_size and every ld * elem_size
 * multiples of 16 (refused before any CUDA call otherwise). prefix may be NULL when prefix_len = 0.
 * Alignment (bytes) of vr_prefix_rows: prefix 16, rows 16, out 16, cu_rows 4, cu_out 4 */
int vr_prefix_rows(const void* prefix, int64_t ldp, const void* rows, int64_t ldr, void* out, int64_t ldo,
                   const int32_t* cu_rows, const int32_t* cu_out, int32_t batch, int32_t prefix_len, int32_t out_rows,
                   int32_t cols, int32_t elem_size, void* stream);


/* ------------------------------------------------------------------------------------
 * Similarity + top-k: replaces `torch.matmul(Q, D^T)` + `torch.topk` of
 * retriever/dense_retriever.py:25-30 (fp32 scores) and the Python merge loop `:88-92`.
 * The [nq, nd] score matrix is never materialised:
 *   vr_score_filter  : wgmma fp16 GEMM on CTA pairs (256 queries x 256 docs per tile, 128 queries per CTA) with a fused per-row running
 *                      top-16 per (query, doc range); writes `lists = 2*ranges` sorted 16-entry candidate lists per query into
 *                      cand_scores / cand_ids [nq, lists*16] (unused lists: score -inf, id -1; the first score of the LAST
 *                      list slot is scratch - the query's running threshold - and carries id -1);
 *   vr_score_rescore : keeps the max(32, 2k) best candidates by approximate score, rescoring them exactly in fp32, top-k by
 *                      (score desc, id asc), and a proof that nothing dropped (by a list or by the pruning) could belong to
 *                      the top-k (flags[q] = 1 when the proof fails; the caller then reruns that query through
 *                      vr_score_exact + vr_topk_rows).
 * Results are therefore exactly the fp32 top-k. Doc ids returned are `local index + id_offset`.
 * Alignment (bytes) of vr_f32_to_f16_rows: src 16, dst_f16 8
 * Alignment (bytes) of vr_score_filter: q_f16 16, d_f16 16, cand_scores 16, cand_ids 16
 * Alignment (bytes) of vr_score_rescore: d_f32 16
 * Alignment (bytes) of vr_score_exact: d_f32 16
 * ---------------------------------------------------------------------------------- */
int vr_score_ranges(int32_t nq, int64_t nd);   /* sizes the candidate buffers: [nq, ranges*2*16]; host arithmetic only (needs no
                                                * GPU); pass the value on to vr_score_filter / vr_score_rescore unchanged */
int vr_score_list_len(void);                   /* 16 */
/* The filter's work decomposition for (nq, nd), host arithmetic only: out6 = {doc tiles of 256, doc ranges R, 256-query blocks,
 * work items = R * blocks (item i = range i / blocks of query block i % blocks, tiles [T*r/R, T*(r+1)/R)), CTA pairs launched,
 * candidate lists per query (= 2 * vr_score_ranges)}. For tests and capacity planning. */
int vr_score_plan(int32_t nq, int64_t nd, int32_t* out6);
int vr_f32_to_f16_rows(const float* src, int64_t rows, int32_t dim, void* dst_f16, float* norms, float* max_norm,
                       void* stream);          /* norms / max_norm optional; *max_norm must be pre-zeroed */
int vr_score_filter(const void* q_f16, int32_t nq, const void* d_f16, int64_t nd, int32_t dim, int32_t ranges,
                    float* cand_scores, int32_t* cand_ids, void* stream);
int vr_score_rescore(const float* q_f32, int32_t nq, const float* d_f32, int64_t nd, int32_t dim, int32_t ranges,
                     const float* cand_scores, const int32_t* cand_ids, const float* max_doc_norm, int32_t k,
                     int64_t id_offset, float* out_scores, int64_t* out_ids, int32_t* flags, void* stream);
/* plain fp32 scan (small problems, flagged queries): scores [nq, nd], any nq. A score has the same bits as the one
 * vr_score_rescore computes for the same (query, doc) pair (same FMA order and reduction). */
int vr_score_exact(const float* q_f32, int32_t nq, const float* d_f32, int64_t nd, int32_t dim, float* scores, void* stream);
/* top-k of every row of scores [rows, cols]; ids == NULL -> column index (+ id_offset), else ids[row, col]
 * (negative ids are skipped): also the k-way merge of per-shard / per-rank partial top-k lists. */
int vr_topk_rows(const float* scores, const int64_t* ids, int32_t rows, int64_t cols, int32_t k, int64_t id_offset,
                 float* out_scores, int64_t* out_ids, void* stream);
/* Same result for few rows x many columns (single-query retrieval over a large index): `chunks` blocks per row each
 * reduce a column range to a top-k list (pass 1, workspace ws_scores / ws_ids [rows, chunks, k]), then the lists are
 * merged (pass 2). One block per row would scan a 1 M-column row k times on a single SM. */
int vr_topk_rows_chunked(const float* scores, int32_t rows, int64_t cols, int32_t k, int64_t id_offset, int32_t chunks,
                         float* ws_scores, int64_t* ws_ids, float* out_scores, int64_t* out_ids, void* stream);

/* Filtered retrieval: the same operations over a chosen subset of the docs.
 * doc_mask: ceil(nd / 32) uint32 words in device memory, 4-byte aligned; doc i (local index, before id_offset) is
 * eligible when bit (i & 31) of word (i >> 5) is set; bits at or past nd are ignored. An ineligible doc is never a
 * candidate and never a result: the results are those of the plain calls over the eligible docs alone, bit for bit.
 * When fewer than k docs are eligible, a row holds the eligible ones in order and then (-inf, -1), as for k > nd.
 * A NULL or misaligned doc_mask, and ids != NULL together with a mask (the mask indexes columns), are refused before
 * any CUDA call.
 * Alignment (bytes) of vr_score_filter_masked: q_f16 16, d_f16 16, cand_scores 16, cand_ids 16, doc_mask 4
 *   vr_score_filter_masked : vr_score_filter over the eligible docs; the candidate lists hold eligible docs only, so
 *                            vr_score_rescore takes them unchanged and its proof covers the eligible docs;
 *   vr_topk_rows_masked    : vr_topk_rows with ids == NULL and columns (docs) filtered by doc_mask;
 *   vr_topk_rows_chunked_masked : vr_topk_rows_chunked with columns filtered by doc_mask. */
int vr_score_filter_masked(const void* q_f16, int32_t nq, const void* d_f16, int64_t nd, int32_t dim, int32_t ranges,
                           float* cand_scores, int32_t* cand_ids, const uint32_t* doc_mask, void* stream);
int vr_topk_rows_masked(const float* scores, const int64_t* ids, int32_t rows, int64_t cols, int32_t k, int64_t id_offset,
                        float* out_scores, int64_t* out_ids, const uint32_t* doc_mask, void* stream);
int vr_topk_rows_chunked_masked(const float* scores, int32_t rows, int64_t cols, int32_t k, int64_t id_offset,
                                int32_t chunks, float* ws_scores, int64_t* ws_ids, float* out_scores, int64_t* out_ids,
                                const uint32_t* doc_mask, void* stream);

/* Document-level retrieval: the top-k GROUPS (documents) of pages, each scored by its best page.
 * doc_groups [nd] int32: the group of each doc (page), in [0, G). group_offsets [G+1] / group_pages [nd] int32: the same
 * mapping as CSR, pages ascending within a group (a stable sort of doc_groups). The score of a group is the maximum exact
 * fp32 score over its eligible pages (the bits vr_score_exact gives each pair; NaN never selected), its best page the
 * lowest page with that maximum; groups rank by (score desc, best page asc). Outputs per query: out_scores [k] f32,
 * out_pages [k] i64 (best page + id_offset), out_groups [k] i64; a group without an eligible page never appears, and
 * fewer than k groups leave a tail of (-inf, -1, -1). With every page its own group the result equals the page top-k.
 * doc_mask (optional, NULL: every page eligible) has the layout of the _masked calls. A NULL or misaligned doc_groups or
 * CSR array, G <= 0, a workspace too small and nd >= 2^31 are refused before any CUDA call.
 * Alignment (bytes) of vr_score_filter_groups: q_f16 16, d_f16 16, cand_scores 16, cand_ids 16, doc_groups 4, doc_mask 4
 * Alignment (bytes) of vr_score_rescore_groups: d_f32 16, doc_groups 4, group_offsets 4, group_pages 4, doc_mask 4
 *   vr_score_filter_groups  : vr_score_filter with GROUP-DISTINCT lists: a list holds at most one page per group (a page
 *                             of a group already listed replaces that entry only when its score is higher). Every page a
 *                             list dropped is <= that list's tail or <= its own group's entry in that list;
 *   vr_score_rescore_groups : step 1 as vr_score_rescore; then the distinct groups of the kept candidates, in approximate
 *                             order, are FULLY rescored (every eligible page, through the CSR) while their pages fit a
 *                             budget of 4096 per query; the top-k of those groups is certified when
 *                             max(list tails, pruned heads, approximate entries of kept groups not rescored) + eps is
 *                             below the k-th group score, else flags[q] = 1 (rerun through vr_score_exact +
 *                             vr_group_topk_rows). Sound with the lists of any filter (page lists meet the invariant);
 *   vr_group_topk_rows      : the group top-k of dense score rows [rows, nd] (vr_score_exact output), from doc_groups
 *                             alone (an order-independent atomicMax of (score, ~page) keys per (row, group), spread over
 *                             the pages whatever the group sizes); chunks >= 2 spreads each row's groups over `chunks`
 *                             blocks (few rows x many groups), 0 or 1 does not. Workspace of
 *                             vr_group_topk_ws_bytes(rows, G, k, chunks) bytes, 16-byte aligned;
 *   vr_merge_group_topk     : merge of per-rank partial group lists [rows, cols] (score, page, group; page < 0 = empty,
 *                             cols <= 512, i.e. world * k <= 512; larger is refused): the first k distinct groups in
 *                             (score desc, page asc) order. A group's best
 *                             page lies on one rank, whose local top-k holds it whenever the group is in the global
 *                             top-k, so the merge is exact when documents span ranks. */
int vr_score_filter_groups(const void* q_f16, int32_t nq, const void* d_f16, int64_t nd, int32_t dim, int32_t ranges,
                           float* cand_scores, int32_t* cand_ids, const int32_t* doc_groups, const uint32_t* doc_mask,
                           void* stream);
int vr_score_rescore_groups(const float* q_f32, int32_t nq, const float* d_f32, int64_t nd, int32_t dim, int32_t ranges,
                            const float* cand_scores, const int32_t* cand_ids, const int32_t* doc_groups,
                            const int32_t* group_offsets, const int32_t* group_pages, int32_t G, const uint32_t* doc_mask,
                            const float* max_doc_norm, int32_t k, int64_t id_offset, float* out_scores, int64_t* out_pages,
                            int64_t* out_groups, int32_t* flags, void* stream);
int64_t vr_group_topk_ws_bytes(int32_t rows, int32_t G, int32_t k, int32_t chunks);
int vr_group_topk_rows(const float* scores, int32_t rows, int64_t nd, const int32_t* doc_groups, int32_t G,
                       const uint32_t* doc_mask, int32_t k, int64_t id_offset,
                       int32_t chunks, void* ws, int64_t ws_bytes, float* out_scores, int64_t* out_pages, int64_t* out_groups,
                       void* stream);
int vr_merge_group_topk(const float* scores, const int64_t* pages, const int64_t* groups, int32_t rows, int32_t cols, int32_t k,
                        float* out_scores, int64_t* out_pages, int64_t* out_groups, void* stream);

/* Per-query filters: each query of a batch searches its own subset of the docs, in the same one pass over the index.
 * A mask set holds `count` masks of the _masked layout, row by row: doc i (local index, before id_offset) is eligible for
 * mask m when bit (i & 31) of words[m * pitch + (i >> 5)] is set; bits at or past nd are ignored. Query row r uses mask
 * of_query[r], which the caller keeps in [0, count) (the values are in device memory and are not checked); a NULL
 * of_query means every row uses mask 0, so the single doc_mask of the _masked calls is the mask set
 * {doc_mask, ceil(nd / 32), NULL, 1}. Each query's result is that of the _masked call of that query alone with its own
 * mask, bit for bit. words and of_query are device pointers; the struct itself is read on the host during the call.
 * Alignment (bytes) of the vr_doc_masks arrays: words 4, of_query 4
 * Every _masks entry point takes the other pointers with the alignment of its _masked or doc_mask counterpart, and
 * refuses before any CUDA call: masks NULL, words NULL or misaligned, count < 1, pitch < ceil(nd / 32) (nd = cols for
 * the top-k calls), and count > 1 with a NULL of_query; the message names the field.
 *   vr_score_filter_masks         : vr_score_filter_masked with a mask per query; the lists of query q hold q's eligible
 *                                   docs only, so vr_score_rescore takes them unchanged;
 *   vr_score_filter_groups_masks  : vr_score_filter_groups with a mask per query;
 *   vr_score_rescore_groups_masks : vr_score_rescore_groups, each query rescoring its own eligible pages;
 *   vr_topk_rows_masks            : vr_topk_rows_masked, row r of scores filtered by the mask of query r (ids must be NULL);
 *   vr_topk_rows_chunked_masks    : vr_topk_rows_chunked_masked with a mask per row;
 *   vr_group_topk_rows_masks      : vr_group_topk_rows with a mask per row.
 * A call over rows [r0, r0 + n) of a larger batch passes of_query + r0. */
typedef struct {
    const uint32_t* words;     /* [count, pitch] mask words */
    int64_t pitch;             /* words per mask, >= ceil(nd / 32) */
    const int32_t* of_query;   /* [rows]: the mask of each query row, or NULL: mask 0 for every row */
    int32_t count;             /* masks in the set, >= 1 */
} vr_doc_masks;

int vr_score_filter_masks(const void* q_f16, int32_t nq, const void* d_f16, int64_t nd, int32_t dim, int32_t ranges,
                          float* cand_scores, int32_t* cand_ids, const vr_doc_masks* masks, void* stream);
int vr_score_filter_groups_masks(const void* q_f16, int32_t nq, const void* d_f16, int64_t nd, int32_t dim, int32_t ranges,
                                 float* cand_scores, int32_t* cand_ids, const int32_t* doc_groups, const vr_doc_masks* masks,
                                 void* stream);
int vr_score_rescore_groups_masks(const float* q_f32, int32_t nq, const float* d_f32, int64_t nd, int32_t dim, int32_t ranges,
                                  const float* cand_scores, const int32_t* cand_ids, const int32_t* doc_groups,
                                  const int32_t* group_offsets, const int32_t* group_pages, int32_t G,
                                  const vr_doc_masks* masks, const float* max_doc_norm, int32_t k, int64_t id_offset,
                                  float* out_scores, int64_t* out_pages, int64_t* out_groups, int32_t* flags, void* stream);
int vr_topk_rows_masks(const float* scores, const int64_t* ids, int32_t rows, int64_t cols, int32_t k, int64_t id_offset,
                       float* out_scores, int64_t* out_ids, const vr_doc_masks* masks, void* stream);
int vr_topk_rows_chunked_masks(const float* scores, int32_t rows, int64_t cols, int32_t k, int64_t id_offset, int32_t chunks,
                               float* ws_scores, int64_t* ws_ids, float* out_scores, int64_t* out_ids,
                               const vr_doc_masks* masks, void* stream);
int vr_group_topk_rows_masks(const float* scores, int32_t rows, int64_t nd, const int32_t* doc_groups, int32_t G,
                             const vr_doc_masks* masks, int32_t k, int64_t id_offset, int32_t chunks, void* ws,
                             int64_t ws_bytes, float* out_scores, int64_t* out_pages, int64_t* out_groups, void* stream);

/* Candidate lists: each query row scores only the docs of its list, reading those rows and no others.
 * A list set holds `count` lists of local doc ids (before id_offset) in CSR form: list m is ids[offsets[m], offsets[m+1]).
 * Query row r uses list of_query[r], which the caller keeps in [0, count); a NULL of_query means every row uses list 0.
 * A list may be in any order and may repeat an id. offsets, ids and of_query are device pointers; the struct itself is
 * read on the host during the call. A call over rows [r0, r0 + n) of a larger batch passes of_query + r0.
 * Alignment (bytes) of the vr_doc_lists arrays: offsets 8, ids 4, of_query 4 */
typedef struct {
    const int64_t* offsets;    /* [count + 1], offsets[0] = 0, non-decreasing */
    const int32_t* ids;        /* [offsets[count]] local doc ids */
    int32_t count;             /* lists in the set, >= 1 */
    const int32_t* of_query;   /* [rows]: the list of each query row, or NULL: list 0 for every row */
} vr_doc_lists;

/* vr_score_lists: the exact fp32 scores of every query row against the docs of its list, as a padded block
 * [nq, width]: out_scores[r, j] = q_r . d[L(r)[j]] (the bits vr_score_exact gives that pair) and out_ids[r, j] = L(r)[j]
 * for j < |L(r)|, then (-inf, -1). With doc_groups (the group table of the _groups calls), out_groups[r, j] is the group
 * of the entry (-1 for padding); doc_groups and out_groups are both given or both NULL. An id outside [0, nd) is never
 * read and gives (-inf, -1). This is the (scores, ids) input of vr_topk_rows, and with the groups that of
 * vr_merge_group_topk, so a row's page or document top-k over its list equals the masked calls' with a mask of exactly
 * the listed docs (a repeated id is emitted once by both selections). Rows that share a list and sit next to each other
 * (sort the rows by list) read each listed row once per tile of up to 8 queries.
 * *status (a device int32 the caller zeroes) gets bit 1 when a list is longer than width (its first width entries are
 * scored) and bit 2 when an of_query value lies outside [0, count) (the row gets padding only).
 * Refused before any CUDA call, naming the field: lists NULL, offsets or ids NULL or misaligned, count < 1, count > 1
 * with a NULL of_query, a misaligned of_query, width < 1, dim % 4 != 0, nd >= 2^31, and a misaligned pointer below.
 * Alignment (bytes) of the vr_score_lists arguments: q_f32 4, d_f32 16, doc_groups 4, out_scores 4, out_ids 8,
 * out_groups 8, status 4 */
int vr_score_lists(const float* q_f32, int32_t nq, const float* d_f32, int64_t nd, int32_t dim, const vr_doc_lists* lists,
                   int32_t width, const int32_t* doc_groups, float* out_scores, int64_t* out_ids, int64_t* out_groups,
                   int32_t* status, void* stream);

/* Range search: for query row r with threshold t_r (thresholds [nq] f32, never NaN), every eligible doc j with exact
 * score s_rj >= t_r (the bits vr_score_exact gives that pair; NaN scores never qualify), ordered by (score desc, id asc).
 * masks (optional, NULL: every doc) is a mask set as in the _masks calls. Three producers and one ordering step:
 *   vr_score_filter_range  : the wgmma fp16 filter of vr_score_filter with a fixed drop threshold per row,
 *                            thr = t_r - eps(|q_r|, max|d|, dim) rounded toward -inf (eps: the bound of the top-k proof),
 *                            appends every doc with approximate score >= thr to cand_ids [nq, cap] (row r's first
 *                            min(counts[r], cap) entries, in no order). counts [nq] is set by the call; counts[r] > cap
 *                            means the row overflowed (only its first cap slots were written), and a row whose |q|
 *                            (q_norms, e.g. the norms output of vr_f32_to_f16_rows) or *max_doc_norm is not < 65504
 *                            has no bound and is marked overflowed too. Every doc with s >= t is a candidate of a row
 *                            that did not overflow;
 *   vr_score_rescore_range : exact fp32 scores of each row's candidates; those with s >= t_r go to out_scores / out_ids
 *                            [nq, cap] (row r's first kept[r] entries, in no order). Overflowed rows get kept[r] = 0:
 *                            rerun them through vr_score_exact + vr_range_rows;
 *   vr_range_rows          : rows of vr_score_exact output [rows, nd] (row r with threshold thresholds[r] and, with
 *                            masks, the mask of row r): the eligible columns with s >= t, as (score, column) into
 *                            out_scores / out_ids [rows, pitch] (first counts[r] entries, in no order; pitch >= nd);
 *   vr_range_sort          : orders such a region (scores / ids [*, pitch], counts[*]) into CSR rows: call row i sorts
 *                            region row r = row_of[i] (row_of NULL: r = i) by (score desc, id asc) and writes it at
 *                            out_scores / out_ids [out_offsets[r], out_offsets[r] + counts[r]), ids + id_offset. The
 *                            caller keeps every counts[r] <= max_count <= pitch. Up to 4096 entries a row sort in shared
 *                            memory; longer rows need a workspace of vr_range_sort_ws_bytes(rows, max_count) bytes.
 * Every entry refuses, before any CUDA call and naming the argument: a NULL or misaligned pointer, nq, rows or nd out of
 * range (rows <= 65535 for vr_range_rows and vr_range_sort), dim not a positive multiple of 8 (4 for the fp32 calls),
 * cap < 1, pitch < nd, max_count outside [0, pitch], a workspace too small, and a bad mask set.
 * Alignment (bytes) of the vr_score_filter_range arguments: q_f16 16, d_f16 16, thresholds 4, q_norms 4, max_doc_norm 4,
 * counts 4, cand_ids 4
 * Alignment (bytes) of the vr_score_rescore_range arguments: q_f32 4, d_f32 16, thresholds 4, counts 4, cand_ids 4,
 * out_scores 4, out_ids 4, kept 4
 * Alignment (bytes) of the vr_range_rows arguments: scores 4, thresholds 4, out_scores 4, out_ids 4, counts 4
 * Alignment (bytes) of the vr_range_sort arguments: scores 4, ids 4, counts 4, row_of 4, out_offsets 8, out_scores 4,
 * out_ids 8, ws 8 */
int vr_score_filter_range(const void* q_f16, int32_t nq, const void* d_f16, int64_t nd, int32_t dim, const float* thresholds,
                          const float* q_norms, const float* max_doc_norm, const vr_doc_masks* masks, int32_t cap,
                          int32_t* counts, int32_t* cand_ids, void* stream);
int vr_score_rescore_range(const float* q_f32, int32_t nq, const float* d_f32, int64_t nd, int32_t dim,
                           const float* thresholds, int32_t cap, const int32_t* counts, const int32_t* cand_ids,
                           float* out_scores, int32_t* out_ids, int32_t* kept, void* stream);
int vr_range_rows(const float* scores, int32_t rows, int64_t nd, const float* thresholds, const vr_doc_masks* masks,
                  int64_t pitch, float* out_scores, int32_t* out_ids, int32_t* counts, void* stream);
int64_t vr_range_sort_ws_bytes(int32_t rows, int32_t max_count);
int vr_range_sort(const float* scores, const int32_t* ids, int64_t pitch, const int32_t* counts, int32_t rows,
                  const int32_t* row_of, const int64_t* out_offsets, int32_t max_count, int64_t id_offset, void* ws,
                  int64_t ws_bytes, float* out_scores, int64_t* out_ids, void* stream);

/* vr_range_groups: the document form of a range region. scores / ids [rows, pitch] with counts[rows] is a region as
 * vr_score_rescore_range and vr_range_rows write it (ids distinct within a row); doc_groups int32 [nd] gives each page its
 * group (document). Row r of the output region (out_scores / out_ids [rows, pitch], first out_counts[r] entries, in no
 * order) holds one entry per group present in row r: the group's first entry in (score desc, id asc) order (+0 = -0, the
 * lower id wins), carrying that entry's own score bits. Entries with a NaN score, an id outside [0, nd) or a group outside
 * [0, G) are dropped. vr_range_sort then orders the output region (its ids are distinct); the groups of the output come
 * from doc_groups. The caller keeps every counts[r] <= max_count <= pitch (entries past max_count are not read). Two
 * passes over each row against a hash table of P = 2^m >= 2 max_count slots: an atomicMax of the (score order, ~page)
 * key per group, then the entry holding its group's key appends itself. Up to 4096 entries a row the table lives in
 * shared memory (one block per row, 12 P bytes); longer rows need a workspace of vr_range_groups_ws_bytes(rows,
 * max_count) bytes. No allocation and no synchronisation.
 * Refused before any CUDA call, naming the argument: a NULL or misaligned pointer, rows outside [1, 65535], nd outside
 * [1, 2^31 - 1), G < 1, max_count outside [0, pitch] and a workspace too small.
 * Alignment (bytes) of the vr_range_groups arguments: scores 4, ids 4, counts 4, doc_groups 4, out_scores 4, out_ids 4,
 * out_counts 4, ws 8 */
int64_t vr_range_groups_ws_bytes(int32_t rows, int32_t max_count);
int vr_range_groups(const float* scores, const int32_t* ids, int64_t pitch, const int32_t* counts, int32_t rows,
                    int32_t max_count, const int32_t* doc_groups, int64_t nd, int32_t G, void* ws, int64_t ws_bytes,
                    float* out_scores, int32_t* out_ids, int32_t* out_counts, void* stream);

/* vr_select_rows: the top-k of each row by a radix select, in passes over the row whose number does not depend on k
 * (DESIGN §4, "Deep top-k"). The contract of vr_topk_rows / vr_topk_rows_masks / vr_topk_rows_chunked(_masks), with the
 * same result bit for bit: out_scores / out_ids [rows, k] in (score desc, id asc) order (+0 = -0, the id decides; a
 * repeated (score, id) pair emitted once; NaN never selected), ids + id_offset, then (-inf, -1). ids (optional, int64
 * [rows, cols]; a negative id is skipped) and masks (the _masks forms: row r filtered by the mask of query r) are
 * exclusive. The chunked forms spread each row over `chunks` blocks, each writing its chunk's top-k into ws_scores /
 * ws_ids [rows, chunks, k], then select from those lists. Cost: about five reads of each row (four 8-bit digit passes,
 * fewer when a bin settles the boundary, plus the gather; ties split at the boundary add one pass per id byte), and a
 * bitonic sort of the k winners in shared memory (k * 16 bytes). No allocation and no synchronisation.
 * Refused before any CUDA call: a NULL or misaligned pointer, rows < 1, cols outside [1, 2^31), k outside [1, 4096],
 * chunks outside [1, 65535], ids with masks, and a bad mask set.
 * Alignment (bytes) of the vr_select_rows arguments: scores 4, ids 8, ws_scores 4, ws_ids 8, out_scores 4, out_ids 8 */
int vr_select_rows(const float* scores, const int64_t* ids, int32_t rows, int64_t cols, int32_t k, int64_t id_offset,
                   float* out_scores, int64_t* out_ids, void* stream);
int vr_select_rows_masks(const float* scores, const int64_t* ids, int32_t rows, int64_t cols, int32_t k, int64_t id_offset,
                         float* out_scores, int64_t* out_ids, const vr_doc_masks* masks, void* stream);
int vr_select_rows_chunked(const float* scores, int32_t rows, int64_t cols, int32_t k, int64_t id_offset, int32_t chunks,
                           float* ws_scores, int64_t* ws_ids, float* out_scores, int64_t* out_ids, void* stream);
int vr_select_rows_chunked_masks(const float* scores, int32_t rows, int64_t cols, int32_t k, int64_t id_offset,
                                 int32_t chunks, float* ws_scores, int64_t* ws_ids, float* out_scores, int64_t* out_ids,
                                 const vr_doc_masks* masks, void* stream);

/* vr_mmr_select: maximal marginal relevance (DESIGN §4) over given candidates. Query row r has the candidates
 * cand_ids [nq, fetch] (local doc ids, row-major) with relevance scores cand_scores [nq, fetch], in (score desc, id asc)
 * order as vr_topk_rows returns them; the first id outside [0, nd) ends the row's candidates (F' of them) and is never
 * read. lambda [nq] f32 is each row's lambda (1: relevance only, 0: diversity only). sim(a, b) is the fp32 dot product of
 * emb rows a and b with the bits vr_score_exact gives that pair. Pick 1 is candidate 0; pick t >= 2 is the unpicked
 * candidate j with the largest v_j = fl(fl(lambda * s_j) - fl(mu * r_j)), mu = fl(1 - lambda), r_j = the maxNum of
 * sim(c_j, e) over the picked e (NaN ignored); NaN ranks below every number and equal values (+0 = -0) go to the lower
 * position. out_scores / out_ids [nq, k] hold the min(k, F') picks in pick order, (s_j, id + id_offset), then (-inf, -1).
 * One thread-block cluster per row holds the row's candidate rows in shared memory (each read from HBM once): the
 * smallest of 1, 2, 4, 8 CTAs whose ceil(fetch / C) rows take at most 144 KiB each, chosen from fetch and dim alone (the
 * bits do not depend on it); each CTA also keeps a copy of the latest pick's row. No allocation and no synchronisation:
 * the call can be captured in a CUDA graph.
 * Refused before any CUDA call, naming the argument: a NULL or misaligned pointer, nq outside (0, 2^28), nd < 1, dim not
 * a positive multiple of 4, fetch outside [1, 128], fetch * dim > 128 * 2304, no cluster size whose share fits 144 KiB,
 * or a share that does not fit 200 KiB with the pick's row (dims of 2304 and less always fit; see
 * visrag_b200.retriever.mmr_fetch_max), and k outside [1, fetch]. lambda's values are the caller's to check (visrag_b200.retriever.mmr_select refuses NaN and
 * values outside [0, 1]).
 * Alignment (bytes) of the vr_mmr_select arguments: emb 16, cand_scores 4, cand_ids 8, lambda 4, out_scores 4,
 * out_ids 8 */
int vr_mmr_select(const float* emb, int64_t nd, int32_t dim, const float* cand_scores, const int64_t* cand_ids, int32_t nq,
                  int32_t fetch, const float* lambda, int32_t k, int64_t id_offset, float* out_scores, int64_t* out_ids,
                  void* stream);

/* vr_group_pages_topm: the m best eligible pages of given groups (documents), the stage of the capped top-k and the
 * inner hits (DESIGN §4). For query row r and slot j < kg, with g = groups[r, j] (int64 [nq, kg], e.g. the out_groups of
 * the _groups calls), the pages of g come from the group CSR of the _groups calls (group_offsets [G+1], group_pages);
 * those eligible under masks (optional, NULL: every page; a mask set as in the _masks calls, row r using the mask of
 * query row r) are scored exactly (the bits vr_score_exact gives each pair; NaN never selected) and the first m by
 * (score desc, page asc) go to out_scores / out_pages [nq, kg, pieces, m] as (score, page + id_offset), then (-inf, -1).
 * A group longer than `piece` pages is split: piece y of (r, j) covers its pages [y piece, (y + 1) piece), and the
 * caller keeps pieces * piece >= the largest group (pages beyond are not read). With pieces > 1, vr_topk_rows over rows
 * nq * kg and cols pieces * m reduces the pieces of each (r, j) to the group's m best. A g < 0 or >= G is empty:
 * padding only, no page is read (a sharded rank passes global groups it does not hold). One block per (r, j, piece), a
 * warp per page, the query row in shared memory. No allocation and no synchronisation: the call can be captured in a
 * CUDA graph.
 * Refused before any CUDA call, naming the argument: a NULL or misaligned pointer, nq < 1, nd outside [1, 2^31), dim not
 * a positive multiple of 4, kg < 1, nq * kg >= 2^31, G < 1, m outside [1, 256], piece outside [1, 4096], pieces outside
 * [1, 65535], dim * 4 + piece * 8 bytes beyond 200 KiB of shared memory, and a bad mask set.
 * Alignment (bytes) of the vr_group_pages_topm arguments: q_f32 4, d_f32 16, groups 8, group_offsets 4, group_pages 4,
 * out_scores 4, out_pages 8 */
int vr_group_pages_topm(const float* q_f32, int32_t nq, const float* d_f32, int64_t nd, int32_t dim, const int64_t* groups,
                        int32_t kg, const int32_t* group_offsets, const int32_t* group_pages, int32_t G,
                        const vr_doc_masks* masks, int32_t m, int32_t piece, int32_t pieces, int64_t id_offset,
                        float* out_scores, int64_t* out_pages, void* stream);

/* Hybrid retrieval (DESIGN §4, "Hybrid retrieval"): the dense score fused with an external score v >= 0 per (query, page),
 * e.g. BM25 over the pages' OCR text. A hit list is CSR over query rows: row r's hits are hit_ids (local pages, distinct
 * within a row) / hit_values [hit_offsets[r], hit_offsets[r + 1]), hit_offsets int64 [rows + 1].
 *
 * vr_fuse_rows: the candidate row of each query, ready for vr_select_rows / vr_topk_rows (which give the (score desc,
 * id asc) order and the k cut). dense_scores / dense_ids [rows, kd] are the dense top-kd of each row in (score desc,
 * id asc) order as vr_select_rows writes it (local ids, a (-inf, -1) tail allowed). Row r of out_scores / out_ids
 * [rows, width] holds slots [0, kd) the dense entries whose page is not a hit of row r ((-inf, -1) for the others), slot
 * kd + i hit i, then (-inf, -1). mode VR_FUSE_SUM: hit i scores fl(hit_dense[r * hit_pitch + i] + fl(weight * v)), with
 * hit_dense the hits' exact dense scores (vr_score_lists' out_scores, hit i at column i), and a dense entry keeps its
 * score; the top-k of the row is the exact top-k of the fused score over the whole index when kd >= k (every listed page
 * scores at least its dense score). mode VR_FUSE_RRF: reciprocal rank fusion, fl(1/fl(c + rank_dense) + 1/fl(c + rank_ext))
 * with c = rrf_c, rank_dense = slot + 1 in the dense window and rank_ext = i + 1 (the caller orders each row's hits by
 * (value desc, id asc)); a missing rank contributes 0; hit_values and hit_dense are not read (may be NULL). The dense
 * entries are hashed in shared memory (2^m >= 2 kd slots), so any hit list length takes the same path. A row with more
 * than width - kd hits keeps its first width - kd and ORs 1 into *status. Repeated hits, negative or non-finite values
 * are the caller's to refuse (visrag_b200.retriever.score_topk_hybrid does, on the host). No allocation and no
 * synchronisation.
 * Refused before any CUDA call, naming the argument: a NULL or misaligned pointer, a mode other than VR_FUSE_SUM /
 * VR_FUSE_RRF, rows < 1, kd outside [1, 4096], width outside [kd, 2^31), hit_pitch < 1 (SUM), weight negative, NaN or
 * infinite (SUM), rrf_c < 0 (RRF).
 * Alignment (bytes) of the vr_fuse_rows arguments: dense_scores 4, dense_ids 8, hit_offsets 8, hit_ids 4, hit_values 4,
 * hit_dense 4, out_scores 4, out_ids 8, status 4
 *
 * vr_group_pages_fused: the document form. vr_group_pages_topm with m = 1 (same traversal, same arguments, same output
 * layout [nq, kg, pieces, 1]) where an eligible page p that is a hit of row r is ranked by fl(s + fl(weight * v)): each
 * (row, slot, piece) gets its best page by fused score (score desc, page asc). Row r's hits must be sorted by id (each
 * page is looked up by a binary search). Reducing the pieces with vr_topk_rows (k = 1) gives each document's fused score
 * and best page. Refused before any CUDA call as vr_group_pages_topm, plus NULL or misaligned hit pointers and a weight
 * that is negative, NaN or infinite.
 * Alignment (bytes) of the vr_group_pages_fused arguments: q_f32 4, d_f32 16, groups 8, group_offsets 4, group_pages 4,
 * hit_offsets 8, hit_ids 4, hit_values 4, out_scores 4, out_pages 8 */
#define VR_FUSE_SUM 0
#define VR_FUSE_RRF 1
int vr_fuse_rows(const float* dense_scores, const int64_t* dense_ids, int32_t rows, int32_t kd, const int64_t* hit_offsets,
                 const int32_t* hit_ids, const float* hit_values, const float* hit_dense, int64_t hit_pitch, int32_t mode,
                 float weight, int32_t rrf_c, int64_t width, float* out_scores, int64_t* out_ids, int32_t* status,
                 void* stream);
int vr_group_pages_fused(const float* q_f32, int32_t nq, const float* d_f32, int64_t nd, int32_t dim, const int64_t* groups,
                         int32_t kg, const int32_t* group_offsets, const int32_t* group_pages, int32_t G,
                         const vr_doc_masks* masks, const int64_t* hit_offsets, const int32_t* hit_ids,
                         const float* hit_values, float weight, int32_t piece, int32_t pieces, int64_t id_offset,
                         float* out_scores, int64_t* out_pages, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VISRAG_B200_H */
