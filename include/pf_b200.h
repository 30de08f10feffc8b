/* pf_b200.h — C-ABI of libpf_b200.so: the sm_90a (Hopper) kernels behind the Pyramid-Flow sampler hot path.
 *
 * Boundary contract:
 *   - plain C, raw device pointers + sizes + a cudaStream_t (passed as void*); no torch types;
 *   - every function returns 0 on success, <0 on error; pf_last_error() gives the message;
 *   - the caller owns every buffer; kernels are stream-ordered and hold no global mutable state;
 *   - there is NO CPU fallback: on a machine without an sm_90 GPU every compute entry fails.
 *
 * Each entry cites the reference op site (file:line under jy0205/Pyramid-Flow @3040d71) it replaces.
 * Abbreviations: F = pyramid_dit/flux_modules/modeling_pyramid_flux.py, B = .../modeling_flux_block.py,
 * N = .../modeling_normalization.py, E = .../modeling_embedding.py, P = pyramid_dit/pyramid_dit_for_video_gen_pipeline.py,
 * S = diffusion_schedulers/scheduling_flow_matching.py, C = video_vae/modeling_causal_conv.py,
 * R = video_vae/modeling_resnet.py, K = video_vae/modeling_block.py, D = video_vae/modeling_enc_dec.py,
 * V = video_vae/modeling_causal_vae.py, MB = pyramid_dit/mmdit_modules/modeling_mmdit_block.py.
 * The text-encoder entries cite transformers 5.5 by class and method: T5 = transformers/models/t5/modeling_t5.py,
 * CLIP = transformers/models/clip/modeling_clip.py.
 */
#ifndef PF_B200_H_
#define PF_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PF_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------ misc */
PF_API const char* pf_last_error(void);
PF_API int pf_version(void);
/* 0 if the current CUDA device is sm_90 (H100) and the driver exposes cuTensorMapEncodeTiled; <0 otherwise. */
PF_API int pf_device_check(void);
/* Loads every kernel instantiation of the library on the CURRENT device and sets its dynamic shared-memory attribute, so
 * that no later launch initialises anything host-side (required before capturing launches into a CUDA graph; also what makes
 * a second GPU driven from the same process work).  Idempotent, thread-safe. */
PF_API int pf_warmup(void);
/* Library options: data-path choices that do not change results (same arithmetic, same bits) but are A/B-measured. */
enum {
  PF_OPT_GEMM_STAGED_RESID = 0, /* GATE_RESID epilogue of the 128-row GEMM kernels: residual read-modify-write by whole row
                                 * segments (a warp per row) instead of one thread per row.  No effect on the 256 x 128 cluster
                                 * kernel, whose epilogue works from the accumulator fragments. */
  PF_OPT_GEMM_WAVE_TILING = 1,  /* with few rows, take the 128 x 128 or 128 x 64 GEMM kernel instead of the 256 x 128 cluster
                                 * kernel when its wave count x tile area, over its measured relative rate, is smaller */
  /* q-tile grouping hints of pf_attn_fwd_masked.  The sm_90a build has one attention kernel (one q tile per CTA, scores in
   * registers); the three keys are accepted and stored so that existing callers keep working, and change nothing. */
  PF_OPT_ATTN_PAIR_KERNEL = 2,
  PF_OPT_ATTN_TILE_PHASE = 3,
  PF_OPT_ATTN_TRIPLE_KERNEL = 4,
  PF_OPT_COUNT = 5
};
#define PF_OPT_DEFAULT_GEMM_STAGED_RESID 1
#define PF_OPT_DEFAULT_GEMM_WAVE_TILING 1
#define PF_OPT_DEFAULT_ATTN_PAIR_KERNEL 1
#define PF_OPT_DEFAULT_ATTN_TRIPLE_KERNEL 1
#define PF_OPT_DEFAULT_ATTN_TILE_PHASE 800
PF_API int pf_set_option(int key, int value);
PF_API int pf_get_option(int key);
/* number of kernels launched by this library since load (bench.py's gpu_launches claim). */
PF_API int64_t pf_launch_count(void);

/* ------------------------------------------------------------------ step contexts (pf_ctx_*, pf_dit_step_*)
 * A pf_ctx owns ONE recorded launch sequence: between pf_ctx_record_begin and pf_ctx_record_end every pf_* launch issued on
 * `stream` by the calling thread is recorded instead of executed (descriptor validation, tensor-map encoding and kernel
 * selection happen once, at record time); pf_dit_step_flux / pf_dit_step_mmdit / pf_vae_decode_chunk then re-issue the whole
 * sequence with one call, on any stream.  What the sequence is -- the ~280 launches of PyramidFluxTransformer.forward
 * (F:392-542) at one (plan, shapes), of PyramidDiffusionMMDiT.forward (M:420-497), or one temporal chunk of
 * CausalVaeDecoder.forward (D:302-366) -- is whatever the host recorded; the three entry points are the same replay under the
 * names of the reference functions they stand for.  The caller owns every buffer the recorded launches point to and must
 * keep them alive and at the same addresses; peer-memory barriers (pf_peer_barrier) may be part of the sequence.
 * pf_ctx_record_end returns the number of recorded launches (>= 0) or < 0 on error. */
typedef struct pf_ctx pf_ctx;
PF_API int pf_ctx_create(pf_ctx** out);
PF_API int pf_ctx_destroy(pf_ctx* ctx);
PF_API int pf_ctx_record_begin(pf_ctx* ctx, void* stream);
PF_API int pf_ctx_record_end(pf_ctx* ctx);
PF_API int pf_ctx_replay(pf_ctx* ctx, void* stream);
PF_API int pf_dit_step_flux(pf_ctx* ctx, void* stream);
PF_API int pf_dit_step_mmdit(pf_ctx* ctx, void* stream);
PF_API int pf_vae_decode_chunk(pf_ctx* ctx, void* stream);

/* ------------------------------------------------------------------ peer memory (sequence parallel over NVLink / NVSwitch)
 * Replaces the reference's all-to-all at the attention boundary (trainer_misc/communicate.py:7-24, called at
 * modeling_flux_block.py:285-295, 314-321, 535-560) and its contiguous()/cat copies: producers store straight into the owning
 * rank's buffer through mapped peer pointers (pf_gemm_desc.peer_qkv, pf_attn_desc.peer_out); pf_peer_barrier orders those
 * stores against their consumers.  One process per GPU on one node; buffers come from pf_peer_alloc (cudaMalloc + CUDA IPC). */
#define PF_MAX_PEERS 8
typedef struct PfPeerGroup {
  void* ptr[PF_MAX_PEERS]; /* one mapped pointer per group member (ptr[my_index] = the local buffer) */
  int32_t n;               /* members */
  int32_t my_index;
} PfPeerGroup;
PF_API int pf_peer_alloc(int64_t bytes, void** ptr);   /* zero-filled device memory that peers can map */
PF_API int pf_peer_free(void* ptr);
PF_API int pf_peer_export(void* ptr, void* handle64);  /* 64-byte CUDA IPC handle of a pf_peer_alloc buffer */
PF_API int pf_peer_open(const void* handle64, void** peer_ptr);
PF_API int pf_peer_close(void* peer_ptr);
/* Barrier over the group: grp->ptr[i] = member i's flag array (PF_MAX_PEERS uint32, zero-initialised, peer memory);
 * epoch_counter = one uint32 in local device memory, advanced by the kernel (graph-replay safe).  Everything this rank's
 * earlier kernels stored to peers is visible to a peer's kernels launched after ITS matching barrier. */
PF_API int pf_peer_barrier(const PfPeerGroup* grp, uint32_t* epoch_counter, void* stream);
/* dst->ptr[i][dst_offset_bytes ...] = src[0 .. bytes) for every member (16-byte granularity). */
PF_API int pf_peer_bcast(const PfPeerGroup* dst, const void* src, int64_t bytes, int64_t dst_offset_bytes, void* stream);

/* ------------------------------------------------------------------ GEMM (wgmma + TMA)
 * out = epilogue(A[rows, K] . W[N, K]^T + bias).  bf16 operands, fp32 accumulation in registers.
 * Replaces every nn.Linear on the DiT path: x_embedder/context_embedder F:290,F:401; to_q/k/v, add_*_proj B:816-835;
 * to_out/to_add_out B:868-872; FeedForward B:73-100; proj_mlp/proj_out B:923-938; norm_out+proj_out F:538-539;
 * with the elementwise ops around them fused into the epilogue (bias, GELU-tanh, per-head RMSNorm N:66-79,
 * RoPE B:34-39, gate*x + residual B:1019-1039).
 *
 * A is addressed as [batches][rows_per_batch][K] (row stride lda); only rows [row_begin, row_begin+row_count) of each
 * batch are computed (the text / video ranges of the joint sequence).  Output row of (b, m) is
 * b*out_batch_rows + out_row_begin + m.
 */
enum {
  PF_EPI_STORE_BF16 = 0, /* out_bf16 = acc + bias                                         */
  PF_EPI_GELU_BF16 = 1,  /* out_bf16 = gelu_tanh(acc + bias)          (diffusers GELU, B:73-75) */
  PF_EPI_STORE_F32 = 2,  /* out_f32  = acc + bias                     (embedders into the fp32 residual stream) */
  PF_EPI_GATE_RESID = 3, /* out_f32 += gate[b, n] * (acc + bias)      (B:1019-1020, 1027-1028, 1032-1039, 937-938) */
  PF_EPI_QKV_ROPE = 4,   /* N = 3*H*hd: bias, RMSNorm(q,k) per head, RoPE(q,k); head-major Q/K/V stores */
  PF_EPI_QKV_GELU = 5,   /* N = 3*H*hd + n_mlp: columns < n_split as QKV_ROPE, the rest as GELU_BF16 (single block, B:923-936) */
  /* text encoders (appended; 0-5 keep their meaning) */
  PF_EPI_GEGLU_BF16 = 6,      /* T5 T5DenseGatedActDense.forward with gelu_new: W = wi_0 and wi_1 interleaved in 64-row blocks,
                               * so in every 128-column tile column j < 64 is the gate and j + 64 the linear term;
                               * out_bf16[r, out_col_begin + tile*64 + j] = gelu_tanh(gate + bias) * (lin + bias).  The output is
                               * n/2 wide.  Requires n % 128 == 0; never runs on the 128 x 64 kernel (kernel_variant 2 is refused). */
  PF_EPI_QUICK_GELU_BF16 = 7, /* out_bf16 = x * sigmoid(1.702 x), x = acc + bias  (CLIP-L hidden_act "quick_gelu", CLIPMLP.forward) */
  PF_EPI_GELU_ERF_BF16 = 8    /* out_bf16 = 0.5 x (1 + erf(x / sqrt 2))            (CLIP-G hidden_act "gelu", CLIPMLP.forward) */
};

typedef struct pf_gemm_desc {
  const void* a; /* bf16 */
  int64_t lda;   /* elements between rows of A */
  int32_t batches, rows_per_batch, row_begin, row_count;
  const void* w; /* bf16 [n, k] row-major (nn.Linear.weight) */
  int32_t n, k;
  const float* bias; /* fp32 [n] or NULL */
  int32_t epilogue;
  /* generic output (STORE_*, GELU, GATE_RESID, and the GELU half of QKV_GELU) */
  void* out;
  int64_t ldo;
  int32_t out_batch_rows, out_row_begin, out_col_begin;
  /* GATE_RESID: fp32 gate[b*gate_batch_stride + n] */
  const float* gate;
  int64_t gate_batch_stride;
  /* QKV_*: outputs bf16 [batches, heads, seq_len, head_dim]; position of (b, m) is out_row_begin + m */
  void* q_out;
  void* k_out;
  void* v_out;
  const float* rope;     /* fp32 [seq_len, head_dim/2, 2] = (cos, sin) per rotation pair, or NULL (no rotation) */
  const float* q_norm_w; /* fp32 [head_dim] */
  const float* k_norm_w; /* fp32 [head_dim] */
  float norm_eps;
  int32_t heads, head_dim, seq_len;
  int32_t n_split; /* QKV_GELU: first n_split (=3*H*hd) columns are q|k|v */
  int32_t kernel_variant; /* 0 = auto; 1 = force the 256 x 128 two-CTA cluster kernel (n % 128 == 0); 2 = force the 128 x 64
                           * kernel.  Same bits either way (same K order, same epilogue arithmetic); exists so tests can pin
                           * each kernel. */
  /* QKV_ROPE under sequence parallelism (peer_count > 1): head h of this rank's token chunk is stored into rank
   * (h / peer_heads)'s buffer peer_qkv[h / peer_heads], laid out [3 (q,k,v)][peer_heads][peer_seq][head_dim], at sequence
   * position peer_row0 + (out_row_begin + m).  q_out/k_out/v_out are ignored.  batches must be 1; every peer_qkv[i] is
   * 16-byte aligned. */
  void* peer_qkv[PF_MAX_PEERS];
  int32_t peer_count, peer_heads, peer_seq, peer_row0;
} pf_gemm_desc;

PF_API int pf_gemm_bf16(const pf_gemm_desc* desc, void* stream);

/* ------------------------------------------------------------------ FP8 (e4m3) GEMM and its quantisers (opt-in)
 * Numerical contract.  e4m3 = float8_e4m3fn: max finite 448, round to nearest even, saturating (F2FP.SATFINITE.E4M3).
 *   Quantising a row x[0..K) (activations: one scale per token; weights: one scale per output channel, the same formula):
 *     amax = max_k |x[k]|;  inv = amax > 0 ? 448.f / amax : 0.f (IEEE fp32 division);  q[k] = e4m3(x[k] * inv);
 *     scale = amax / 448.f.  A row of zeros gives zeros and scale 0; no NaN or Inf.  |x[k] * inv| <= 448 (1 + 2^-23), which
 *     rounds to 448, so a host restatement that casts with torch (which does not saturate) gives the same bits.
 *   GEMM:  acc[r, n] = sum_k q_a[r, k] q_w[n, k] in fp32, then y = acc * scale_a[r] * scale_w[n] + bias[n], and y goes into
 *     the epilogue exactly as in pf_gemm_bf16 (every PF_EPI_*).  Hopper's fp8 wgmma adds into its accumulator with reduced
 *     internal precision, so the kernel adds the partial sum of every K = 128 slice into the fp32 accumulator separately
 *     (promotion); the sum order depends on K only (a row's outputs do not depend on the launch's row range).
 *
 * pf_gemm_fp8: the pf_gemm_bf16 descriptor with d->a, d->w pointing to e4m3 data (lda counts elements = bytes);
 * a_row_scale fp32 [batches, rows_per_batch] indexed like A's rows, w_col_scale fp32 [n].  Requires n % 128 == 0,
 * k % 16 == 0, lda % 16 == 0, kernel_variant 0 and no peer stores (peer_count 0).  The text-encoder epilogues (6-8) are
 * bf16 only: pf_gemm_fp8 refuses them. */
PF_API int pf_gemm_fp8(const pf_gemm_desc* desc, const float* a_row_scale, const float* w_col_scale, void* stream);
/* pf_ln_modulate with an e4m3 output: the fp32 LN-modulated row is quantised directly (one rounding) with the contract above;
 * y_fp8 row stride = dim; row_scale fp32 [batches, rows_per_batch] (rows outside the range are not written). */
PF_API int pf_ln_modulate_fp8(const float* x, void* y_fp8, float* row_scale, int32_t batches, int32_t rows_per_batch,
                              int32_t row_begin, int32_t row_count, int32_t dim, const float* shift, const float* scale,
                              int64_t mod_batch_stride, float eps, void* stream);
/* Row quantiser: bf16 x[r, 0..cols) (row stride ldx) -> e4m3 y[r, ...] (row stride ldy) + row_scale[r], for the rows
 * r = b * rows_per_batch + row_begin + m, m < row_count.  cols % 8 == 0, ldx % 8 == 0, ldy % 8 == 0, 16-byte aligned x and
 * 8-byte aligned y. */
PF_API int pf_quantize_rows_fp8(const void* x_bf16, int64_t ldx, void* y_fp8, int64_t ldy, float* row_scale, int32_t batches,
                                int32_t rows_per_batch, int32_t row_begin, int32_t row_count, int32_t cols, void* stream);

/* ------------------------------------------------------------------ masked joint attention (wgmma + TMA)
 * softmax(Q K^T * scale + mask) V with mask(q, kv) = (seg[q] == seg[kv]) && (time[q] >= time[kv])  (F:318-350),
 * replacing F.scaled_dot_product_attention with the dense bool mask at B:363-365 and B:596-598.
 * q,k,v: bf16 [batch, heads, seq, 64]; out: bf16 [batch, seq, heads*64] with row stride ldo (elements).
 * seg/time: int32 [batch, seq].  tile_sched: int32, built by pf_attn_build_schedule (host) from seg/time.
 */
typedef struct pf_attn_desc {
  const void* q;
  const void* k;
  const void* v;
  void* out;
  int64_t ldo;
  int32_t batch, heads, seq, head_dim;
  float scale;
  const int32_t* seg;        /* device [batch, seq] */
  const int32_t* time;       /* device [batch, seq] */
  const int32_t* tile_sched; /* device; layout documented at pf_attn_build_schedule */
  int32_t sched_stride;      /* int32 entries per (batch, q_tile) row */
  int32_t variant;           /* 0 = default.  0x10 / 0x20 additionally require the pair / group schedule below; 1 / 2 / 3 are
                              * accepted.  Every value runs the same kernel (pf_attn.cu) and gives the same bits. */
  int32_t q_row_begin;       /* only q rows >= q_row_begin are computed (multiple of 128; 0 = all).  The last single block
                              * needs the current clip's rows only (history outputs are discarded, reference F:380). */
  const int32_t* pair_sched; /* device; built by pf_attn_build_pair_schedule from tile_sched, same sched_stride.  Part of a
                              * caller's plan; the kernel works from tile_sched and reads none of the pair / group arrays. */
  const int32_t* pair_mask_index; /* device; from pf_attn_build_pair_masks (required with pair_sched) */
  const void* pair_mask_bits;     /* device; [blocks, 128, 4] uint32 */
  /* sequence parallelism (peer_count > 1, batch 1): row q of this rank's head group is stored into rank
   * (q / peer_chunk_rows)'s buffer peer_out[...] at row q % peer_chunk_rows, columns peer_col_begin + h*64 (row stride ldo);
   * `out` is ignored.  peer_col_begin % 8 == 0, peer_col_begin + heads*64 <= ldo, every peer_out[i] 16-byte aligned. */
  void* peer_out[PF_MAX_PEERS];
  int32_t peer_count, peer_chunk_rows, peer_col_begin;
  /* variant 0x20: schedule and row masks of groups of three
   * q tiles from pf_attn_build_group_schedule / pf_attn_build_group_masks (group = 3), same sched_stride */
  const int32_t* group_sched;
  const int32_t* group_mask_index;
  const void* group_mask_bits;
  /* optional (NULL = not written): fp32 [batch, heads, seq], each row's log-sum-exp of the SCALED scores in natural log,
   * lse[q] = ln sum_kv exp(scale * q.k) over the allowed kv (+inf for a row without one); what pf_attn_bwd_masked takes.
   * Whole local launches only: refused with peer_count > 1 or q_row_begin != 0.  Without it the kernel runs unchanged. */
  float* lse;
} pf_attn_desc;

/* Host helper: from host copies of seg/time ids builds, for each (batch, 128-row q tile), the list of 128-wide kv
 * tiles that contain at least one allowed pair, flagged full (no element mask needed) or partial.
 * Row layout: [count, (kv_tile << 1) | needs_mask, ...].  Returns the number of int32 written per row
 * (sched_stride) or <0 on error.  `out` may be NULL to query the size: stride = 1 + ceil(seq/128). */
PF_API int pf_attn_build_schedule(const int32_t* seg_host, const int32_t* time_host, int32_t batch, int32_t seq,
                                  int32_t* out, int64_t* allowed_pairs /* [batch] or NULL */);
/* Host helper: pairs the q tiles from the end of the sequence (pair p = tiles q_tiles-2-2p and q_tiles-1-2p; the first tile is
 * alone when q_tiles is odd) and merges their kv lists.  Row layout per (batch, pair): [count, entry...], entry =
 * (kv_tile << 4) | flags_lo | (flags_hi << 2), flags = bit0: the tile has an allowed pair in this kv tile, bit1: it needs the
 * element mask (a tile without bit0 is computed fully masked).  `out` holds batch * ceil(q_tiles/2) rows of sched_stride. */
PF_API int pf_attn_build_pair_schedule(const int32_t* tile_sched_host, int32_t batch, int32_t seq, int32_t sched_stride,
                                       int32_t* out);
/* Host helper: the element masks of a pair schedule.  For every (pair entry, tile X) whose flags say "partial" it
 * assigns a block index (mask_index[batch, n_pairs, 2 * sched_stride], entry e / tile X at [2 e + X], -1 otherwise) and, when
 * mask_bits != NULL, fills block = 128 rows x 4 uint32: bit i of word w of row r = q row r of the tile may attend kv column
 * 32 w + i of the kv tile.  Returns the number of blocks needed (call once with mask_bits = NULL to size the buffer). */
PF_API int64_t pf_attn_build_pair_masks(const int32_t* seg_host, const int32_t* time_host, const int32_t* pair_sched_host,
                                        int32_t batch, int32_t seq, int32_t sched_stride, int32_t* mask_index,
                                        uint32_t* mask_bits, int64_t capacity_blocks);
/* Host helpers: the pair forms generalised to groups of `group` (2..4) q tiles counted from the end
 * of the sequence.  Entry = (kv_tile << 8) | flags, 2 flag bits per tile X at bit 2 X (X = 0 the lowest tile of the group);
 * mask_index[batch, n_groups, group * sched_stride], entry e / tile X at [group e + X]; blocks as in the pair form.  With
 * pair_sched_host / pair_mask_index_host (the pair schedule of the same tile_sched) no bits are built: the indices point into
 * the PAIR schedule's block pool (a block depends on (q tile, kv tile) only), mask_bits is ignored, and the return value is
 * the number of pool blocks referenced. */
PF_API int pf_attn_build_group_schedule(const int32_t* tile_sched_host, int32_t batch, int32_t seq, int32_t sched_stride,
                                        int32_t group, int32_t* out);
PF_API int64_t pf_attn_build_group_masks(const int32_t* seg_host, const int32_t* time_host, const int32_t* group_sched_host,
                                         int32_t batch, int32_t seq, int32_t sched_stride, int32_t group,
                                         int32_t* mask_index, uint32_t* mask_bits, int64_t capacity_blocks,
                                         const int32_t* pair_sched_host /* or NULL */,
                                         const int32_t* pair_mask_index_host /* or NULL */);
PF_API int pf_attn_fwd_masked(const pf_attn_desc* desc, void* stream);
/* Host helper: the kv-major transpose of a pf_attn_build_schedule schedule, for the backward's dK / dV pass.  For each
 * (batch, 128-row kv tile) it lists, in increasing order, the q tiles whose row of tile_sched_host names this kv tile, with the
 * same partial flag.  Row layout: [count, (q_tile << 1) | needs_mask, ...], sched_stride int32 per row (the stride of the q
 * schedule, >= 1 + ceil(seq/128)); `out` holds batch * ceil(seq/128) rows. */
PF_API int pf_attn_build_kv_schedule(const int32_t* tile_sched_host, int32_t batch, int32_t seq, int32_t sched_stride,
                                     int32_t* out);

/* ------------------------------------------------------------------ masked joint attention backward (wgmma + TMA)
 * Gradients of out = softmax(Q K^T * scale + mask) V with the mask of pf_attn_fwd_masked, replacing the autograd backward of
 * F.scaled_dot_product_attention with the dense [B,1,S,S] bool mask that the reference's training path runs in every block
 * (VarlenSelfAttentionWithT5Mask B:363-365, VarlenSelfAttnSingle B:596-598; the mask built by merge_input F:341-350).
 * With P = exp(scale * Q K^T - lse) on the allowed pairs (0 elsewhere) and delta[q] = sum_d dO[q, d] O[q, d]:
 *   dV = P^T dO,   dS = P o (dO V^T - delta),   dQ = scale * dS K,   dK = scale * dS^T Q.
 * Three launches, no atomics (the result is deterministic): delta (one warp per row), dK / dV (one CTA per (b, h, kv tile),
 * q tiles streamed in the order of kv_sched) and dQ (one CTA per (b, h, q tile), kv tiles in the order of tile_sched).
 * Operands bf16, every product and sum in fp32; head_dim 64, any seq (rows past seq are neither read as data nor stored). */
typedef struct pf_attn_bwd_desc {
  const void* q;       /* bf16 [batch, heads, seq, 64] */
  const void* k;
  const void* v;
  const void* out;     /* bf16 [batch, seq, heads*64]: the forward's output; row stride ldo, batch stride out_batch_stride */
  int64_t ldo, out_batch_stride;
  const void* dout;    /* bf16 [batch, seq, heads*64]: the gradient of out; row stride lddo, batch stride dout_batch_stride
                        * (a view: e.g. the stage slice of a gradient whose rows hold more than one stage, so its batch stride
                        * is not seq * lddo).  Strides in elements, multiples of 8; row strides >= heads*64. */
  int64_t lddo, dout_batch_stride;
  const float* lse;    /* fp32 [batch, heads, seq] from pf_attn_fwd_masked */
  int32_t batch, heads, seq, head_dim;
  float scale;
  const int32_t* seg;        /* device [batch, seq] */
  const int32_t* time;       /* device [batch, seq] */
  const int32_t* tile_sched; /* device, pf_attn_build_schedule */
  const int32_t* kv_sched;   /* device, pf_attn_build_kv_schedule (same sched_stride) */
  int32_t sched_stride;
  float* delta;              /* workspace fp32 [batch, heads, seq] */
  void* dq;                  /* bf16 [batch, heads, seq, 64] */
  void* dk;
  void* dv;
} pf_attn_bwd_desc;
PF_API int pf_attn_bwd_masked(const pf_attn_bwd_desc* desc, void* stream);

/* ------------------------------------------------------------------ stage pack + RoPE of the training attention
 * One stage's head-major q / k / v for pf_attn_fwd_masked / pf_attn_bwd_masked, replacing the torch glue of the training
 * attention: the stack of q / k / v, the cat of the stage's text rows (encoder rows stage::n_stages) with its video rows, the
 * fp32 apply_rope and transpose(1, 2) (VarlenSelfAttentionWithT5Mask B:342-360 and MB:287-305, VarlenSelfAttnSingle
 * B:580-594; apply_rope B:34-39, MB:271-276).  Packed row s of batch b is text row s of text source row
 * b * n_stages + stage for s < text_len, else video row row0 + s - text_len of batch b.  With freqs, q and k are rotated in
 * fp32 without contraction and rounded once to bf16:
 *   packed[2p + c] = fl(fl(f[b, s, p, c, 0] * x[2p]) + fl(f[b, s, p, c, 1] * x[2p + 1]));
 * v is copied (rounded to bf16).  No accumulation, one launch.
 *
 * pf_attn_stage_pack_bwd is the exact inverse for gradients: it reads the packed gradients (dq, dk, dv in `packed`) and writes
 * the stage's rows of the source gradients (the video / text pointers, in their own dtype and strides), for q and k
 *   d x[2p + j] = fl(fl(g[2p] * f[b, s, p, 0, j]) + fl(g[2p + 1] * f[b, s, p, 1, j]))
 * (what autograd computes through apply_rope's mul / sum_to_size / float()).  Each source row belongs to one stage, so the
 * stages' launches together write every row of the gradients exactly once.
 *
 * Layout rules (checked; a violation returns <0 before any launch): head_dim 64; unit column stride; source strides in elements,
 * positive multiples of 8, base pointers 16-byte aligned; 0 <= row0, row0 + rows <= src_rows; 0 <= stage < n_stages when
 * text_len > 0; freqs 16-byte aligned with strides multiples of 4 and a row stride >= 128. */
typedef struct pf_attn_pack_desc {
  int32_t batch, heads, head_dim;
  int32_t text_len;                /* T; 0 = no text sources (the single blocks' sequence already holds the text) */
  int32_t rows, row0, src_rows;    /* the stage's video rows [row0, row0 + rows) of sources with src_rows rows per batch */
  int32_t n_stages, stage;         /* text source row of batch b: b * n_stages + stage */
  /* video sources [batch, src_rows, heads, 64] and text sources [batch * n_stages, text_len, heads, 64]: q, k, v at [0..2];
   * strides (batch, row, head) in elements; is_f32 1 = fp32, 0 = bf16 */
  void* video[3];
  int64_t video_strides[3][3];
  int32_t video_f32[3];
  void* text[3];
  int64_t text_strides[3][3];
  int32_t text_f32[3];
  const float* freqs;              /* fp32 [batch, text_len + rows, 32, 2, 2] (each row's 128 floats contiguous), or NULL */
  int64_t freqs_batch_stride, freqs_row_stride;
  void* packed[3];                 /* bf16 [batch, heads, text_len + rows, 64] contiguous: q, k, v (or dq, dk, dv) */
} pf_attn_pack_desc;
PF_API int pf_attn_stage_pack(const pf_attn_pack_desc* desc, void* stream);
PF_API int pf_attn_stage_pack_bwd(const pf_attn_pack_desc* desc, void* stream);

/* ------------------------------------------------------------------ varlen pack / unpack of the flash training path
 * The padding-free form of the training attention, replacing the torch glue around flash_attn_varlen_func in
 * VarlenFlashSelfAttentionWithT5Mask (B:189-263; called through FluxAttnProcessor2_0.varlen_flash_attn B:796-798, B:852-857)
 * and VarlenFlashSelfAttnSingle (B:452-516; FluxSingleAttnProcessor2_0 B:736-738, B:772-777), with the per-stage
 * `indices` / `seqlens_in_batch` of merge_input's flash branch (F:295-317).
 *
 * Every stage i of a call site has a padded sequence of stage_len[i] rows per batch (T + L_i: its text rows, then its video
 * rows; the single blocks' sequence already holds the text).  A padded position p enumerates (stage, batch, row) stage-major,
 * then batch, then row: the reference's pad_attention_mask.flatten() of each stage, concatenated.  The call site's sources
 * for (stage i, batch b, row s) are those of pf_attn_stage_pack with stage = i, row0 = stage_row0[i]: text row s of text
 * source row b * n_stages + i when s < text_len, else video row stage_row0[i] + s - text_len of batch b.
 * row_map[r] is the padded position of packed row r, in the order of the reference's torch.cat(qkv_list) (each stage's
 * `indices`, offset by the stage's first padded position); pad_map[p] is the packed row of position p, or -1 for a row the
 * reference drops (padded text).  Both maps live on the device and are trusted: they must be inverse to each other. */
#define PF_ATTN_VARLEN_MAX_STAGES 8
typedef struct pf_attn_varlen_layout {
  int32_t batch, heads, head_dim;
  int32_t text_len;          /* T: rows of each stage's sequence held by the text sources; 0 = no text sources */
  int32_t src_rows;          /* video source rows per batch */
  int32_t n_stages;          /* 1 .. PF_ATTN_VARLEN_MAX_STAGES */
  int32_t stage_len[PF_ATTN_VARLEN_MAX_STAGES];   /* rows of stage i's padded sequence per batch (> text_len) */
  int32_t stage_row0[PF_ATTN_VARLEN_MAX_STAGES];  /* video source row of stage i's row text_len */
  int32_t total;             /* packed rows (the sum of the cu_seqlens lengths) */
  const int32_t* row_map;    /* device int32 [total] */
  const int32_t* pad_map;    /* device int32 [batch * sum(stage_len)] */
} pf_attn_varlen_layout;

/* pf_attn_varlen_pack: packed row r of the head-major bf16 q / k / v [1, heads, total, 64] that pf_attn_fwd_masked /
 * pf_attn_bwd_masked read (batch 1, seq = total) is the source row of row_map[r], with q and k rotated by stage i's table
 * freqs[i] at (b, s) exactly as pf_attn_stage_pack does (fp32, no contraction, one rounding to bf16): the stack / cat /
 * apply_rope (B:34-39) / index_first_axis / torch.cat of B:208-226 and B:468-483, in one launch for every stage.
 * pf_attn_varlen_pack_bwd reads the packed gradients and writes every row of every source gradient exactly once, in the
 * source's dtype and strides: the transposed RoPE of pf_attn_stage_pack_bwd for rows a packed row names, 0 for the others
 * (what autograd gives through index_first_axis).  No atomics.  Sources follow the layout rules of pf_attn_stage_pack. */
typedef struct pf_attn_varlen_pack_desc {
  pf_attn_varlen_layout layout;
  void* video[3];            /* [batch, src_rows, heads, 64]; strides (batch, row, head) in elements; is_f32 1 = fp32 */
  int64_t video_strides[3][3];
  int32_t video_f32[3];
  void* text[3];             /* [batch * n_stages, text_len, heads, 64] (ignored when text_len = 0) */
  int64_t text_strides[3][3];
  int32_t text_f32[3];
  const float* freqs[PF_ATTN_VARLEN_MAX_STAGES];  /* stage i: fp32 [batch, stage_len[i], 32, 2, 2] rows of 128 floats, or NULL */
  int64_t freqs_batch_stride[PF_ATTN_VARLEN_MAX_STAGES], freqs_row_stride[PF_ATTN_VARLEN_MAX_STAGES];
  void* packed[3];           /* bf16 [1, heads, total, 64] contiguous: q, k, v (or dq, dk, dv) */
} pf_attn_varlen_pack_desc;
PF_API int pf_attn_varlen_pack(const pf_attn_varlen_pack_desc* desc, void* stream);
PF_API int pf_attn_varlen_pack_bwd(const pf_attn_varlen_pack_desc* desc, void* stream);

/* pf_attn_varlen_unpack: the attention output [total, heads*64] (bf16, row stride ld_packed) scattered into the call site's
 * outputs, video [batch, src_rows, heads*64] and text [batch * n_stages, text_len, heads*64], each fp32 or bf16: row s of
 * stage i gets packed row pad_map[p], a dropped row gets 0 (pad_input into zeros_like(query) / zeros_like(encoder_query),
 * B:201-202, B:247-258, B:464, B:504-512).  One launch; every output row written once.
 * pf_attn_varlen_unpack_bwd gathers the output gradients (the same pointers, any strides satisfying the rules) into the
 * packed bf16 dout [total, heads*64] that pf_attn_bwd_masked reads, rounding fp32 to bf16.
 * Layout rules (checked): unit column stride; batch and row strides positive multiples of 8 elements, row strides >=
 * heads*64; base pointers 16-byte aligned; ld_packed a multiple of 8, >= heads*64. */
typedef struct pf_attn_varlen_unpack_desc {
  pf_attn_varlen_layout layout;
  void* video;
  int64_t video_strides[2];  /* batch, row */
  int32_t video_f32;
  void* text;                /* ignored when text_len = 0 */
  int64_t text_strides[2];
  int32_t text_f32;
  void* packed;
  int64_t ld_packed;
} pf_attn_varlen_unpack_desc;
PF_API int pf_attn_varlen_unpack(const pf_attn_varlen_unpack_desc* desc, void* stream);
PF_API int pf_attn_varlen_unpack_bwd(const pf_attn_varlen_unpack_desc* desc, void* stream);

/* ------------------------------------------------------------------ LayerNorm + AdaLN modulate pre-pass (HBM-bound)
 * y_bf16[r, :] = LN(x_f32[r, :], eps) * (1 + scale[b, :]) + shift[b, :]   (N:174, N:234, N:120, B:1022-1023, B:1035-1036)
 * rows [row_begin, row_begin+row_count) of each batch of the joint [batches, rows_per_batch, dim] stream.
 */
PF_API int pf_ln_modulate(const float* x, void* y_bf16, int32_t batches, int32_t rows_per_batch, int32_t row_begin,
                          int32_t row_count, int32_t dim, const float* shift, const float* scale,
                          int64_t mod_batch_stride, float eps, void* stream);

/* ------------------------------------------------------------------ small-M linear (HBM-bound GEMV)
 * y[m, n] (+)= act_out( sum_k act_in(x[m, k]) * W[n, k] + bias[n] ), m <= 8; W bf16, x/y fp32.
 * Used for the per-step AdaLN modulation of ALL layers in one launch (N:147,164,209,223,99,110) and the
 * timestep/text conditioning MLPs (E:84-158, E:185-201).  act: 0 none, 1 SiLU.
 */
PF_API int pf_small_linear(const float* x, int32_t m, int32_t k, const void* w_bf16, const float* bias, int32_t n,
                           float* y, int32_t act_in, int32_t act_out, int32_t accumulate, int32_t round_in_bf16,
                           void* stream);

/* sinusoidal timestep embedding, flip_sin_to_cos=True, downscale_freq_shift=0 (E:11-62): out fp32 [m, dim],
 * out[:, :dim/2] = cos(t * f_i), out[:, dim/2:] = sin(t * f_i), f_i = exp(-ln(1e4) * i / (dim/2)); rounded to bf16
 * values when round_bf16 != 0 (E:195).  t is fp32 [m] (already rounded to bf16 by the caller, P:750). */
PF_API int pf_timestep_embedding(const float* t, int32_t m, int32_t dim, float* out, int32_t round_bf16,
                                 void* stream);

/* patchify one clip: latent bf16/fp32 [B, C, T, H, W] -> tokens bf16 [B, tok_begin + (t h w), (p1 p2 c)], p=2 (F:285-286).
 * tokens row stride = 4*C; rows_per_batch = total tokens of all clips of the unit. */
PF_API int pf_patchify(const void* latent, int32_t latent_is_f32, int32_t b, int32_t c, int32_t t, int32_t h, int32_t w,
                       void* tokens_bf16, int32_t rows_per_batch, int32_t tok_begin, void* stream);
/* unpatchify: x fp32 [B, rows_per_batch, 4*C] rows [row_begin, +t*h/2*w/2) -> out [B, C, T, H, W] (F:383-387). */
PF_API int pf_unpatchify(const float* x, int32_t rows_per_batch, int32_t row_begin, int32_t b, int32_t c, int32_t t,
                         int32_t h, int32_t w, void* out, int32_t out_is_f32, void* stream);

/* fused CFG combine + Euler step (P:771-776, S:278-286):
 * v = vu + g*(vc - vu); x_out = x + dsigma * v.  v: fp32 [2, n] (uncond, cond); x fp32 [n]. */
PF_API int pf_cfg_euler_step(const float* v2, float guidance, float dsigma, const float* x, float* x_out, int64_t n,
                             void* stream);
/* Stage hop of generate_one_unit (P:729-743) in one kernel: nearest x2 up-sampling of the latent planes x [planes, h, w]
 * (bf16 or fp32), block noise of sample_block_noise (P:697-703: each 2x2 block ~ N(0, (1+gamma) I - gamma 11^T)) formed as L z
 * from iid normals z [planes, 2h, 2w] (fp32, drawn on the device) with L = chol16 (host, row-major lower-triangular 4x4), and
 * the renoise  out = alpha * up(x) + beta * noise.  Opt-in on the host side: same distribution as the reference's python loop
 * of MultivariateNormal.sample() calls, different RNG consumption. */
PF_API int pf_stage_hop(const void* x, int32_t x_is_f32, const float* z, void* out, int64_t planes, int32_t h, int32_t w,
                        float alpha, float beta, const float* chol16, void* stream);

/* ------------------------------------------------------------------ causal 3-D convolution (VAE decode, wgmma + TMA)
 * Replaces CausalConv3d -> nn.Conv3d (C:46-146), kernel 3x3x3 or 1x1x1, stride 1, on channels-last bf16 activations.
 * x: [B, T + kt - 1, H, W, Cin]: the (kt-1) causal-padding frames are physically present in front (zeros for the first
 * chunk, the previous chunk's last input frames afterwards = the reference's feature cache C:126-143); spatial zero
 * padding is implicit (TMA out-of-bounds fill).  wgt: bf16 [Cout, kt*kh*kw*Cin], K index = tap*Cin + ci with
 * tap = (dt*kh + dh)*kw + dw (re-laid out once at weight import).  Cin and Cout must be multiples of 64 (pad).
 * store_mode: 0 plain [B, out_t_total, H, W, out_c] at frame t + out_t_offset (+ optional bf16 residual, R:148);
 *             1 spatial depth-to-space 'b (c p1 p2) t h w -> b c t (h p1) (w p2)' (CausalUpsample2x R:616);
 *             2 temporal depth-to-space 'b (c p) t h w -> b c (t p) h w' at frame 2t + p + out_t_offset, frames < 0
 *               dropped (CausalTemporalUpsample2x R:724-727 with is_init_image => out_t_offset = -1).
 */
typedef struct pf_conv3d_desc {
  const void* x;
  int32_t b, t, h, w, cin; /* OUTPUT frames / height / width (= input dims at unit stride) */
  const void* wgt;
  const float* bias; /* fp32 [cout] or NULL */
  int32_t cout, kt, kh, kw;
  int32_t store_mode;
  void* out;
  int32_t out_f32; /* plain mode output type: 0 = bf16, 1 = fp32, 2 = uint8 image clamp(v*127.5+127.5, 0, 255) (decode_latent, P:1238) */
  int32_t out_t_total, out_t_offset, out_c;
  int32_t store_channels; /* first store_channels conv outputs are stored (the rest is filter padding) */
  const void* residual;   /* bf16 [B, res_t_total, H, W, out_c] read at frame t + res_t_offset, plain mode only */
  int32_t res_t_total, res_t_offset;
  int32_t stride_t, stride_h, stride_w; /* 0/1 = unit stride; 2 = the encoder's down-samplers (C:66-67: CausalDownsample2x
                                         * stride (1,2,2) R:322, CausalTemporalDownsample2x stride (2,1,1) R:486).  b,t,h,w
                                         * stay OUTPUT dims; x is [B, (t-1)*stride_t + kt, h*stride_h, w*stride_w, cin]. */
  int32_t kernel_variant; /* 0 = auto; 1 = 128-wide filter tiles (cout % 128 == 0); 2 = 64-wide filter tiles.
                           * Both accumulate in the same K order: the choice never changes the bits. */
} pf_conv3d_desc;
PF_API int pf_causal_conv3d(const pf_conv3d_desc* desc, void* stream);

/* ------------------------------------------------------------------ causal 3-D convolution backward (VAE training)
 * Autograd of CausalConv3d.forward with temporal_chunk=False (C:116-126: F.pad(x, (1,1,1,1,2,0)) -> nn.Conv3d(padding=0),
 * stride 1, (1,2,2) or (2,1,1)), which the reference's VAE training step (train/train_video_vae.py) runs through cuDNN.
 *
 * pf_conv3d_pack: src [b, c, t, h, w] (bf16 or fp32, element strides `strides`, so contiguous and channels_last_3d tensors
 * are read in place) -> dst channels-last bf16 [b, t_total, h*dil_h, w*dil_w, cpad]; src voxel (t, h, w) lands at
 * (t_offset + t*dil_t, h*dil_h, w*dil_w), every other element of dst (causal frames, inserted zeros, channels >= c) is
 * written as zero.  Forward form: t_offset = kt-1, dilations 1 -- pf_causal_conv3d's x.  Gradient form: dy at t_offset 0,
 * dilated by the conv's stride, t_total = T_in + kt - 1: the input of the data gradient (see pf_conv3d_wgrad) and the dy
 * pf_conv3d_wgrad reads.  bias_grad (fp32 [c], or NULL): the sum of src over (b, t, h, w), from fp32 per-row partial sums
 * added in an order fixed by the shape (workspace >= (b*t*h + min(b*t*h, 128)) * cpad floats); dy is read once for both.
 *
 * The data gradient has no entry of its own: it is pf_causal_conv3d at stride 1 over the dilated grid, on the packed dy
 * (t = T_in, h = H_in, w = W_in, cin = Cout padded), with the filter flipped on all three axes and Cin / Cout swapped
 * (wgt [Cin_pad, taps*Cout_pad], same tap-major K order), store_channels = out_c = Cin:
 *   time: dx[s] = sum_e dy_up[s + e] W[2-e]^T;  space: dx[i] = sum_e dy_up[i + e - 1] W[2-e]^T  (dy_up = dy with zeros
 *   inserted along a strided axis, plus kt-1 zero frames at the end because the causal padding is in front). */
typedef struct pf_conv3d_pack_desc {
  const void* src;
  int32_t src_f32;
  int32_t b, c, t, h, w;
  int64_t strides[5]; /* element strides of src's (b, c, t, h, w) */
  void* dst;
  int32_t cpad, t_total, t_offset;
  int32_t dil_t, dil_h, dil_w; /* 1 or 2 */
  float* bias_grad;
  float* workspace;
  int64_t workspace_floats;
} pf_conv3d_pack_desc;
PF_API int pf_conv3d_pack(const pf_conv3d_pack_desc* desc, void* stream);
/* pf_conv3d_wgrad: dw fp32 [cout_real, cin_real, kt, kh, kw] (PyTorch's Conv3d weight layout) =
 *   sum over output voxels v of dy[v, co] * x_pad[v * stride + tap, ci]
 * x: the forward's packed input, bf16 [b, (t-1)*stride_t + kt, h*stride_h, w*stride_w, cin]; dy: the packed gradient, bf16
 * [b, dy_t_total, h*stride_h, w*stride_w, cout] with output voxel (t, h, w) at (t*stride_t, h*stride_h, w*stride_w) (read
 * through TMA element strides, so the data gradient's dilated buffer serves both).  b, t, h, w are OUTPUT dims; cin / cout
 * are the padded channel counts (multiples of 64).  The voxel range is split in a number of parts that depends on the shape
 * only; each part's fp32 partial goes to `workspace` (pf_conv3d_wgrad_workspace floats, at most 2^26 unless one part
 * alone is larger) and the parts are added in a fixed order: deterministic, no atomics. */
typedef struct pf_conv3d_wgrad_desc {
  const void* x;
  const void* dy;
  int32_t dy_t_total;
  int32_t b, t, h, w;
  int32_t cin, cout, cin_real, cout_real;
  int32_t kt, kh, kw;
  int32_t stride_t, stride_h, stride_w;
  float* dw;
  float* workspace;
  int64_t workspace_floats;
} pf_conv3d_wgrad_desc;
/* floats of workspace pf_conv3d_wgrad needs for this descriptor's shape (< 0 if the descriptor is invalid) */
PF_API int64_t pf_conv3d_wgrad_workspace(const pf_conv3d_wgrad_desc* desc);
PF_API int pf_conv3d_wgrad(const pf_conv3d_wgrad_desc* desc, void* stream);

/* per-frame GroupNorm (CausalGroupNorm C:36-43) on channels-last bf16 [frames, voxels, channels]:
 * stats[frame, group] = (mean, rstd); workspace: >= frames * 64 * channels * 2 floats.  Deterministic, and independent of
 * how many frames are passed per call (chunk-invariant).  Per-channel sums are taken in fp32 about the frame's first voxel
 * and combined in double, so a large group mean does not cancel the variance: mean within 1e-5 std + 2^-23 |mean| and
 * rstd within 1e-5 relative of an fp64 two-pass GroupNorm of the same bf16 input, at |mean|/std up to 100 and frames
 * up to 768x1280 voxels. */
PF_API int pf_groupnorm_stats(const void* x_bf16, int32_t frames, int64_t voxels, int32_t channels, int32_t groups,
                              float eps, float* stats, float* workspace, int64_t workspace_floats, void* stream);
/* y[b, t + y_t_offset, vox, c] = act((x[b, t, vox, c] - mean) * rstd * gamma[c] + beta[c]), act = SiLU if silu
 * (R:127-129, R:139-141, D:362-363); y has y_t_total frames per batch (room for the next conv's causal halo). */
PF_API int pf_groupnorm_apply(const void* x_bf16, void* y_bf16, int32_t b, int32_t t, int64_t voxels, int32_t channels,
                              int32_t groups, const float* stats, const float* gamma, const float* beta, int32_t silu,
                              int32_t y_t_total, int32_t y_t_offset, void* stream);
/* ------------------------------------------------------------------ trainable GroupNorm (+ SiLU) (VAE training)
 * Autograd of CausalGroupNorm.forward (C:36-43: GroupNorm of every (batch, frame) over (channels of a group) x H x W) and of
 * the SiLU after it (CausalResnetBlock3D norm1 -> nonlinearity R:127-129, norm2 -> nonlinearity R:139-141, the encoder's /
 * decoder's conv_norm_out -> conv_act D:194-195, D:362-363), which the reference's VAE training step runs as torch's
 * group_norm + silu in fp32 under autocast.
 *
 * x: [b, c, t, h, w], bf16 or fp32, element strides x_strides, read in place in one of two forms (strides of size-1 axes
 * are ignored): channel form, channels_last_3d (c stride 1, w stride c, h stride w*c; b and t strides multiples of 8 and
 * x 16-byte aligned), or plane form (w stride 1, h stride w: every (b, c, t) plane contiguous, any b / c / t strides, e.g.
 * NCDHW).  Any other layout is refused.  c % 8 == 0, c % groups == 0, c <= 2048; gamma, beta fp32 [c].
 * pf_groupnorm_train_fwd: stats fp32 [b*t, groups, 2] = (mean, rstd) (kept for the backward);
 *   y = act((x - mean) * rstd * gamma + beta) (act = SiLU if silu), bf16 or fp32 (y_f32), dense in x's form:
 *   channels-last [b, t, h, w, c] for channel form, [b, c, t, h, w] for plane form.  For a bf16 channel-form x, stats and
 *   a bf16 y are bit-identical to pf_groupnorm_stats + pf_groupnorm_apply (the same device code).
 * pf_groupnorm_train_bwd: dy (bf16 or fp32, dy_f32) in x's form, any strides of that form; with z = xhat*gamma + beta
 *   recomputed and dz = dy * SiLU'(z) (or dy): dbeta = sum dz, dgamma = sum dz*xhat (fp32 [c], either may be NULL) and
 *   dx = rstd * (gamma dz - mean(gamma dz) - xhat mean(gamma dz xhat)) (means per frame and group) in x's dtype, dense in
 *   x's form (NULL: not computed).  x and dy are read twice (once for dx), dx written once.
 * Both need a workspace of pf_groupnorm_train_workspace floats (per (frame, split, channel) fp32 partial sums); the split
 * count depends on h*w only, there are no atomics: the bits depend on the shape alone. */
typedef struct pf_groupnorm_train_desc {
  const void* x;
  int32_t x_f32;
  int32_t b, c, t, h, w;
  int64_t x_strides[5]; /* element strides of x's (b, c, t, h, w) */
  int32_t groups;
  float eps;
  int32_t silu;
  const float* gamma;
  const float* beta;
  float* stats;         /* [b*t, groups, 2]: written by the forward, read by the backward */
  void* y;              /* forward output */
  int32_t y_f32;
  const void* dy;       /* backward input */
  int32_t dy_f32;
  int64_t dy_strides[5];
  void* dx;             /* backward outputs */
  float* dgamma;
  float* dbeta;
  float* workspace;
  int64_t workspace_floats;
} pf_groupnorm_train_desc;
/* floats of workspace the forward and the backward need for this descriptor's shape (< 0 if the descriptor is invalid) */
PF_API int64_t pf_groupnorm_train_workspace(const pf_groupnorm_train_desc* desc);
PF_API int pf_groupnorm_train_fwd(const pf_groupnorm_train_desc* desc, void* stream);
PF_API int pf_groupnorm_train_bwd(const pf_groupnorm_train_desc* desc, void* stream);
/* in-place row softmax of bf16 scores [rows, ld]: softmax over the first `cols` columns of scale*s, zeros in the padding
 * (mid-block attention, diffusers Attention used at K:454-460). */
PF_API int pf_softmax_rows(void* s_bf16, int64_t rows, int32_t cols, int64_t ld, float scale, void* stream);
/* latent [B, C, T, H, W] -> channels-last bf16 [B, y_t_total, H, W, cpad] at frame t + y_t_offset, channels >= C zero,
 * optional per-frame affine z*scale[t] + shift[t] (decode_latent's un-normalisation, P:1226-1230). */
PF_API int pf_pack_latent(const void* z, int32_t z_is_f32, int32_t b, int32_t c, int32_t t, int32_t h, int32_t w,
                          void* y_bf16, int32_t cpad, int32_t y_t_total, int32_t y_t_offset, const float* frame_scale,
                          const float* frame_shift, void* stream);
/* Cross-fade of neighbouring decoded tiles (blend_v / blend_h, V:397-407), tensors viewed as fp32 [outer, L, inner] with L the
 * blended axis: b[o, y, i] = a[o, la - extent + y, i] * (1 - y/extent) + b[o, y, i] * (y/extent) for y < extent (in place). */
PF_API int pf_blend_tiles(const float* a, float* b, int64_t outer, int32_t la, int32_t lb, int64_t inner, int32_t extent,
                          void* stream);

/* ------------------------------------------------------------------ text encoders (T5 v1.1 encoder, CLIP text transformer)
 * The GEMMs run on pf_gemm_bf16: the packed q|k|v projection and CLIPTextModelWithProjection's text_projection on
 * STORE_BF16, the residual adds after the attention output projection and the MLP down-projection on GATE_RESID with a ones
 * gate into an fp32 residual stream, the MLP up-projection on GEGLU (T5) / QUICK_GELU (CLIP-L) / GELU_ERF (CLIP-G).  CLIP's
 * LayerNorms (CLIPEncoderLayer.forward, CLIPTextTransformer.forward final_layer_norm) run on pf_ln_modulate with
 * shift = bias, scale = weight - 1 and mod_batch_stride = 0.
 *
 * Short-sequence attention: T5Attention.forward (scores + position_bias + the T5Stack.forward additive key mask, fp32
 * softmax) and CLIPAttention.forward (causal, scale head_dim^-0.5):
 *   out[b, q, h*64 + :] = softmax_k(scale * Q[b,q,h] . K[b,k,h] + bias[h, k - q + seq - 1] + mask(b, q, k)) . V[b,k,h]
 *   mask = -inf where key_mask[b, k] == 0 (for every query row, padded rows included, as under T5's additive mask),
 *          or causal && k > q.
 * qkv: bf16 [batch * seq, ld_qkv], q of head h at columns [64 h, +64), k at 64 (heads + h), v at 64 (2 heads + h) (the packed
 * QKV GEMM output).  out: bf16 [batch * seq, ldo].  bias: fp32 [heads, 2 seq - 1] (T5Attention.compute_bias as a Toeplitz
 * table) or NULL; key_mask: int32 [batch, seq] or NULL.  seq <= 256, head_dim 64.  A batch whose key mask is all zeros has
 * no defined result (the host wrapper refuses it); such a row is written as zeros. */
typedef struct pf_attn_text_desc {
  const void* qkv;
  int64_t ld_qkv;
  void* out;
  int64_t ldo;
  int32_t batch, heads, seq, head_dim;
  float scale;
  const float* bias;
  const int32_t* key_mask;
  int32_t causal;
} pf_attn_text_desc;
PF_API int pf_attn_fwd_text(const pf_attn_text_desc* desc, void* stream);
/* T5LayerNorm.forward: y_bf16[r, :] = x[r, :] * rsqrt(mean(x[r, :]^2) + eps) * w  (w fp32 [dim]), for rows
 * [row_begin, row_begin + row_count) of each batch of x fp32 [batches, rows_per_batch, dim]; y has x's row layout. */
PF_API int pf_rms_norm_rows(const float* x, void* y_bf16, const float* w, int32_t batches, int32_t rows_per_batch,
                            int32_t row_begin, int32_t row_count, int32_t dim, float eps, void* stream);
/* Embedding lookup (T5Stack.forward embed_tokens, no scaling; CLIPTextEmbeddings.forward token + position):
 * out_f32[r, :] = table[ids[r], :] (+ pos_table[r % rows_per_batch, :]), ids int32 [rows], table bf16 [vocab, dim], pos_table
 * bf16 [max_pos, dim] or NULL.  The host validates ids against vocab; the kernel never reads outside the table (an id out of
 * range gives a zero row). */
PF_API int pf_embed_tokens(const int32_t* ids, int64_t rows, int32_t rows_per_batch, const void* table, int32_t vocab,
                           int32_t dim, const void* pos_table, int32_t max_pos, float* out_f32, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* PF_B200_H_ */
