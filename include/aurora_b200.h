/*
 * aurora_b200.h — C ABI of libaurora_b200.so: the sm_90a (Hopper) kernels behind Aurora's forward pass.
 *
 * The reference (microsoft/aurora) is pure Python/PyTorch and has no FFI; its seam is the Python
 * module boundary (Aurora.forward, aurora/model/aurora.py:265).  Every entry point below replaces a
 * group of ATen/cuBLAS/cuDNN/SDPA calls made by one reference function, cited as file:line relative
 * to the reference checkout.  INTEGRATION.md shows the ctypes binding a maintainer would add.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes, no C++/torch types.
 *   - Every pointer is a DEVICE pointer owned by the caller (PyTorch allocates everything); the
 *     library never allocates device memory and keeps no pointer after a call returns.
 *   - `stream` is a cudaStream_t passed as void*; all work is enqueued on it, nothing synchronises.
 *   - Return value: 0 (AB_OK) or a negative AbStatus; ab_last_error() gives a thread-local message.
 *   - bf16 tensors are raw uint16 storage (torch.bfloat16); "f32" is IEEE float.
 *   - Row-major everywhere; `ld*` are leading dimensions in ELEMENTS.
 */
#ifndef AURORA_B200_H_
#define AURORA_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define AB_ABI_VERSION 2

typedef enum AbStatus {
  AB_OK = 0,
  AB_ERR_INVALID_ARGUMENT = -1,
  AB_ERR_CUDA = -2,
  AB_ERR_UNSUPPORTED = -3
} AbStatus;

/* ABI version of the loaded library (AB_ABI_VERSION it was built with). */
int ab_version(void);

/* Thread-local description of the last failing call ("" if none). */
const char* ab_last_error(void);

/* Number of kernels this library has launched since load (all threads); bench.py reports the delta
 * over the timed region as `gpu_launches`. */
unsigned long long ab_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * Dense projections — replaces every nn.Linear on the path:
 *   swin3d.py:153 (qkv), :169 (proj), :61-64 (MLP fc1 + GELU, fc2), :554 (PatchMerging reduction),
 *   :609,:612 (PatchSplitting lin1/lin2), perceiver.py:141-152 (to_q/to_kv/to_out), :79-84 (MLP),
 *   patchembed.py:112 (conv3d with kernel==stride, i.e. a GEMM), decoder.py:214,250 (heads).
 *
 *   out[m, n] = act( sum_k A[m, k] * W[n, k] + bias[n] ) + residual[m, n]
 *
 * A: bf16|fp16 [M, K] (lda), W: same type [N, K] (ldw; nn.Linear layout), fp32 accumulation in registers
 * (wgmma.mma_async, TMA-staged 128B-swizzled operand tiles).  bias (f32 [N]) and residual
 * (f32 [M, ldr]) are optional (NULL).  act: AB_ACT_NONE or AB_ACT_GELU_ERF (exact erf GELU, as
 * nn.GELU()).  Either or both outputs may be requested: out_f32 [M, ld_f32], out_bf16 [M, ld_bf16].
 * Requirements: K % 8 == 0, lda % 8 == 0, ldw % 8 == 0, A/W 16-byte aligned.
 * ---------------------------------------------------------------------------------------------- */
enum { AB_ACT_NONE = 0, AB_ACT_GELU_ERF = 1 };

/* 16-bit storage / tensor-core operand types.  The Swin backbone uses bf16 (the reference's autocast
 * recipe, aurora.py:327-343); encoder and decoder, which the reference keeps in fp32, use fp16 operands
 * (11-bit mantissa, same wgmma rate, saturating stores) to stay closer to it. */
enum { AB_DT_BF16 = 0, AB_DT_F16 = 1 };

struct AbHaloPush; /* declared below */

typedef struct AbGemm {
  const void* a;       /* bf16 [M, K] */
  const void* w;       /* bf16 [N, K] */
  const float* bias;   /* f32 [N] or NULL */
  const float* residual; /* f32 [M, ldr] or NULL */
  float* out_f32;      /* f32 [M, ld_f32] or NULL */
  void* out_bf16;      /* bf16 [M, ld_bf16] or NULL */
  int32_t m, n, k;
  int32_t lda, ldw, ldr, ld_f32, ld_bf16;
  int32_t act;
  int32_t in_dtype;    /* AB_DT_*: type of a and w */
  int32_t out_dtype;   /* AB_DT_*: type of the 16-bit output ("out_bf16") */
  /* Optional fused exchange (latitude-sharded forecast): the epilogue ALSO stores the boundary rows this descriptor
   * names — columns [tok_off, tok_off + tok_bytes) of the first / last rows of every level of the [C, rows, W, N]
   * output — straight into the neighbouring GPUs' halo slots over NVLink and publishes the round like ab_halo_push
   * (which it replaces for this exchange; `local` is ignored).  16-bit-only bf16 output; at least one row to send. */
  const struct AbHaloPush* peer_push;
} AbGemm;

int ab_gemm_bf16(const AbGemm* g, void* stream);


/* ------------------------------------------------------------------------------------------------
 * 3-D shifted-window attention — replaces, for one Swin3DTransformerBlock (swin3d.py:440-509):
 *   torch.roll (:472,:501), pad_3d / crop_3d (:482,:497), window_partition_3d / window_reverse_3d
 *   (:485,:494), compute_3d_shifted_window_mask (:303-360), maybe_adjust_windows (util.py:53-71) and
 *   F.scaled_dot_product_attention (:164,:166).
 *
 * qkv : bf16 [batch*C*H*W, 3*D], the QKV projection of the FLAT token stream (row = (c*H + h)*W + w,
 *       columns [q | k | v], each head-major with head_dim 64: the layout nn.Linear(D, 3D) produces).
 * out : bf16 [batch*C*H*W, D], heads merged, written at the source token of every window position.
 * `window`/`shift` are the CONFIGURED sizes (e.g. {2,6,12} / {1,3,6} or {0,0,0}); clamping to the
 * resolution, two-sided zero padding, the cyclic shift and the 0/-100 group mask (only when shifted;
 * `warped` merges the left/right longitude groups) are computed in-kernel.  Zero-padded positions
 * take q|k|v from pad_qkv (bf16 [3*D] = the projection bias, because x = 0 there) and are attended to
 * exactly as the reference does in unshifted blocks.  `bias` is an optional dense additive term
 * f32 [num_heads, N, N] (N = tokens per window); NULL for every shipped Aurora checkpoint.
 * ---------------------------------------------------------------------------------------------- */
typedef struct AbWindowAttention {
  const void* qkv;
  const void* pad_qkv; /* bf16 [3*D]; required when the window grid is zero-padded */
  void* out;
  const float* bias;   /* optional, usually NULL */
  int32_t batch;
  int32_t res[3];      /* C, H, W */
  int32_t window[3];
  int32_t shift[3];
  int32_t num_heads;
  int32_t head_dim;    /* must be 64 */
  int32_t warped;
  /* Latitude slab (one forecast sharded over GPUs along H; all zero = whole grid).  qkv / out then hold only the
   * token rows [slab_h_begin, slab_h_begin + slab_h_rows) of the GLOBAL (C, H, W) grid, level-major
   * [C, slab_h_rows, W, .], batch must be 1; `halo_kv` bf16 [2, C, slab_halo, W, 2*D] holds the K | V columns of
   * the slab_halo rows above ([0]: rows h_begin-halo .. h_begin-1) and below ([1]: rows h_end .. h_end+halo-1) the
   * slab, cyclic in H (received from the neighbouring ranks; queries of foreign rows are never needed, and only
   * the rows that windows touching the slab actually reach have to be valid).  Every window touching the slab is
   * computed, only the slab's own rows are written.  slab_halo >= window[1] - 1; full 144-token windows only. */
  int32_t slab_h_begin, slab_h_rows, slab_halo;
  int32_t reserved_;
  const void* halo_kv;
  /* Peer-memory transport: control words of this rank's halo buffer (AbHaloPush.ctrl) or NULL.  When given, the kernel
   * itself waits for both neighbours' pushes of the current round — just before its first foreign row, interior windows
   * run first — and ab_halo_wait must NOT be enqueued separately.  NULL: halo_kv is complete when the kernel starts. */
  const uint32_t* halo_ctrl;
} AbWindowAttention;

int ab_window_attention(const AbWindowAttention* p, void* stream);

/* Window bookkeeping of one block: number of windows per batch element, tokens per (clamped) window
 * and whether the group mask applies.  Host-only, no launch. */
int ab_window_geometry(const int32_t res[3], const int32_t window[3], const int32_t shift[3],
                       int32_t* n_windows, int32_t* n_tokens, int32_t* shifted);

/* Test hook: materialise the in-kernel index arithmetic.  idx_out int32 [n_windows*n_tokens] receives
 * the source token of every window position (-1 = zero padding), group_out uint8 the mask group id
 * (27 = padding).  Must equal roll -> pad -> window_partition_3d / compute_3d_shifted_window_mask. */
int ab_window_index_map(const int32_t res[3], const int32_t window[3], const int32_t shift[3], int32_t warped,
                        int32_t* idx_out, uint8_t* group_out, void* stream);

/* The same function evaluated on the host (HOST pointers): the index arithmetic is one
 * __host__ __device__ routine (csrc/window_index.cuh), so this pins it without a GPU. */
int ab_window_index_map_host(const int32_t res[3], const int32_t window[3], const int32_t shift[3],
                             int32_t warped, int32_t* idx_out, uint8_t* group_out);

/* ------------------------------------------------------------------------------------------------
 * Latitude-sharded forecast: halo exchange through peer memory (NVLink / NVSwitch), no NCCL on the step path.
 * The reference has no multi-GPU forward (SURVEY 8e); the exchange exists because the shifted windows of
 * swin3d.py:470-503 straddle the latitude bands.  See csrc/halo.cu for the protocol.
 *
 * Every rank allocates ONE device buffer (PyTorch owns it): AB_HALO_CTRL_BYTES of control words followed by
 * 2 (parity) x 2 (side: 0 = rows above the band, 1 = rows below) slots of C * halo * W * tok_bytes each, zero-filled
 * once.  ab_ipc_export makes it mappable by the neighbouring processes, ab_ipc_open maps a neighbour's buffer
 * (peer access is enabled on first use), ab_ipc_close unmaps it.
 * ---------------------------------------------------------------------------------------------- */
#define AB_IPC_HANDLE_BYTES 64
#define AB_HALO_CTRL_BYTES 256

/* handle: AB_IPC_HANDLE_BYTES bytes to send to the peer process; offset: of dev_ptr inside its allocation. */
int ab_ipc_export(const void* dev_ptr, uint8_t* handle, uint64_t* offset);
/* Map the allocation behind `handle` (exported by ANOTHER process on this node); *base_out + offset is the
 * peer's dev_ptr in this process's address space. */
int ab_ipc_open(const uint8_t* handle, void** base_out);
int ab_ipc_close(void* base);

typedef struct AbHaloPush {
  const void* local;     /* this rank's band, [C, rows, W, src_tok_bytes] contiguous (qkv: src_tok_bytes = 3D * 2) */
  void* above_slot;      /* PEER address: side-1 slot (current parity) of the rank above, [C, slot_rows, W, tok_bytes] */
  void* below_slot;      /* PEER address: side-0 slot (current parity) of the rank below */
  uint32_t* above_flag;  /* PEER address: control word 1 ("rows below me have landed") of the rank above */
  uint32_t* below_flag;  /* PEER address: control word 0 ("rows above me have landed") of the rank below */
  uint32_t* ctrl;        /* this rank's own control words (start of its buffer) */
  int32_t c, rows, w;
  int32_t slot_rows;     /* rows a slot holds per level (the halo capacity, window height - 1) */
  int32_t rows_to_above; /* my FIRST rows the rank above needs: land in its slot rows [0, n) */
  int32_t rows_to_below; /* my LAST rows the rank below needs: land in its slot rows [slot_rows - n, slot_rows) */
  int64_t src_tok_bytes; /* bytes per token of `local` */
  int64_t tok_off_bytes; /* byte range of every token that is sent: [tok_off_bytes, tok_off_bytes + tok_bytes) */
  int64_t tok_bytes;     /* (k | v of the qkv projection: offset D * 2, length 2D * 2); all multiples of 16 */
} AbHaloPush;

/* Copy the first / last rows of every level of `local` into the neighbours' slots and publish the round. */
int ab_halo_push(const AbHaloPush* p, void* stream);
/* Block the stream until BOTH neighbours' pushes of the current round have landed in this rank's slots.  (The window
 * attention kernel does this itself when it is given AbWindowAttention.halo_ctrl; this stand-alone wait serves other
 * consumers and tests.) */
int ab_halo_wait(uint32_t* ctrl, void* stream);

/* ------------------------------------------------------------------------------------------------
 * LayerNorm + modulation + residual, one pass over the token stream:
 *
 *   out[r, :] = residual[rr, :] + LN(y[r, :]) * scale + shift + add_rows[r % add_mod, :]
 *
 * Replaces AdaptiveLayerNorm + the residual adds of a Swin block (film.py:48-49, swin3d.py:507-508:
 * scale = scale_bias + scale(c), shift = shift(c), both precomputed vectors), the post-res-norm of the
 * Perceiver blocks (perceiver.py:225-232: scale/shift = LayerNorm affine, residual = latents broadcast
 * with rr = (r / res_div) % res_mod) and the encoder's surface MLP residual plus position / scale /
 * time embeddings (encoder.py:320, 344-363: add_rows).  LN statistics in fp32, eps as given.
 * y: bf16 [rows, ld_y]; scale/shift: f32 [dim] or NULL (1 / 0); residual: f32 or NULL; res_mod == 0 means
 * rr = r.  Outputs: f32 and/or bf16, may alias `residual` (each row is read before it is written) and
 * out_bf16 may alias `y`.  dim % 8 == 0, dim <= 2048.
 * ---------------------------------------------------------------------------------------------- */
typedef struct AbLnModResidual {
  const void* y;
  const float* scale;
  const float* shift;
  const float* residual;
  const float* add_rows;
  float* out_f32;
  void* out_bf16;
  int64_t rows;
  int64_t res_div, res_mod;
  int64_t add_mod;
  int32_t dim;
  int32_t ld_y, ld_res, ld_f32, ld_bf16;
  float eps;
  int32_t in_dtype;   /* AB_DT_*: type of y */
  int32_t out_dtype;  /* AB_DT_*: type of out_bf16 */
} AbLnModResidual;

int ab_ln_mod_residual(const AbLnModResidual* p, void* stream);

/* ------------------------------------------------------------------------------------------------
 * One whole Swin3DTransformerBlock (swin3d.py:440-509) in place on the token stream: qkv projection, [halo
 * exchange of a latitude slab], shifted-window attention, output projection, adaLN + residual, MLP (erf GELU),
 * adaLN + residual — 8 to 10 launches of this library on `stream`.  See csrc/block.cu.
 *   x_f32   f32 [tokens, dim]   residual stream, updated in place
 *   x_b16   bf16 [tokens, dim]  16-bit copy of the stream (A operand of qkv / fc1), rewritten after each sub-layer
 *   out_b16 optional: where the 16-bit copy of the block OUTPUT goes instead of x_b16 (leading dimension
 *           ld_out_b16, AB_DT_* out_b16_dtype), e.g. one half of the decoder's [x | skip] concatenation
 *   weights bf16 in nn.Linear layout [out, in] (LoRA merged by the caller), biases / modulation vectors f32;
 *           scale = scale_bias + scale(c), shift = shift(c) of AdaptiveLayerNorm (film.py:48-49)
 *   workspace: ab_swin_block_workspace_bytes(tokens, dim, hidden) bytes, 256-byte aligned, owned by the caller
 *   res / window / shift as in AbWindowAttention.  Latitude slab (slab_h_rows > 0): `res[1]` is the GLOBAL height,
 *   the stream holds rows [slab_h_begin, +slab_h_rows); halo_kv as in AbWindowAttention; halo_push (optional) is
 *   the peer-memory exchange to run between the projection and the attention (its `local` is filled in here).
 * ---------------------------------------------------------------------------------------------- */
typedef struct AbSwinBlock {
  float* x_f32;
  void* x_b16;
  void* out_b16;
  const void* w_qkv;
  const void* w_proj;
  const void* w_fc1;
  const void* w_fc2;
  const float* b_qkv;
  const float* b_proj;
  const float* b_fc1;
  const float* b_fc2;
  const void* pad_qkv;   /* bf16 [3 * dim]: the qkv bias, q | k | v of zero-padded tokens */
  const float* scale1;
  const float* shift1;
  const float* scale2;
  const float* shift2;
  void* workspace;
  const struct AbHaloPush* halo_push;
  const void* halo_kv;
  int32_t dim, hidden, num_heads;
  int32_t res[3], window[3], shift[3];
  int32_t ld_out_b16, out_b16_dtype;
  int32_t slab_h_begin, slab_h_rows, halo_rows;
  float eps;
  int32_t fuse_ln;  /* != 0: adaLN + residual in the epilogue of proj / fc2 (ab_gemm_ln_residual) where dim allows */
  int32_t fuse_push; /* != 0: the QKV projection's epilogue pushes the halo rows itself (AbGemm.peer_push) */
} AbSwinBlock;

int ab_swin_block_workspace_bytes(int64_t tokens, int32_t dim, int32_t hidden, size_t* bytes);
int ab_swin_block(const AbSwinBlock* b, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Projection with AdaptiveLayerNorm + residual fused into its epilogue (swin3d.py:507-508 with film.py:48-49):
 *
 *   out[m, :] = residual[m, :] + LN( A[m, :] · W^T + bias ) * scale + shift
 *
 * = ab_gemm_bf16 followed by ab_ln_mod_residual, in one kernel: the projection output never goes to HBM (the
 * statistics are taken on the fp32 accumulator in registers).  A cluster of CTAs owns whole rows, so N is fixed
 * to 512 or 1024 (ab_gemm_ln_supported).  A, W: bf16|fp16 [M, K] / [N, K]; bias, scale, shift: f32 [N] or NULL
 * (0 / 1 / 0); residual f32 [M, ldr] or NULL; outputs f32 [M, ld_f32] (may alias residual) and / or 16-bit
 * [M, ld_16].  LN without affine, biased variance, eps as given.
 * ---------------------------------------------------------------------------------------------- */
typedef struct AbGemmLn {
  const void* a;
  const void* w;
  const float* bias;
  const float* scale;
  const float* shift;
  const float* residual;
  float* out_f32;
  void* out_16;
  int32_t m, n, k;
  int32_t lda, ldw, ldr, ld_f32, ld_16;
  int32_t in_dtype, out_dtype; /* AB_DT_* */
  float eps;
} AbGemmLn;

int ab_gemm_ln_supported(int32_t n);
int ab_gemm_ln_residual(const AbGemmLn* p, void* stream);

/* ------------------------------------------------------------------------------------------------
 * A whole stage in ONE call: ab_run_ops executes a caller-built list of operations in order on `stream` — e.g. the
 * complete Swin3DTransformerBackbone (swin3d.py:884-936: 48 AB_OP_SWIN_BLOCK + patch merges / splits with their
 * projections), which the engine records once per input signature and then replays with one call per step.  The list
 * is plain host memory owned by the caller (the "plan": it bakes device pointers, so it stays valid as long as the
 * buffers it names do); the library keeps nothing.  Stops at the first failing operation and returns its status.
 * ---------------------------------------------------------------------------------------------- */
enum { AB_OP_GEMM = 1, AB_OP_SWIN_BLOCK = 2, AB_OP_LN_MOD_RESIDUAL = 3, AB_OP_PATCH_MERGE_LN = 4, AB_OP_PATCH_SPLIT_LN = 5 };

typedef struct AbPatchMergeLn { /* arguments of ab_patch_merge_ln */
  const float* x;
  const float* gamma;
  const float* beta;
  void* out_bf16;
  int32_t batch, c, h, w, d;
  float eps;
} AbPatchMergeLn;

typedef struct AbPatchSplitLn { /* arguments of ab_patch_split_ln */
  const void* y_bf16;
  const float* gamma;
  const float* beta;
  void* out_bf16;
  int32_t batch, c, h, w, d, crop_h, crop_w;
  float eps;
} AbPatchSplitLn;

/* PatchMerging3D front half (swin3d.py:526-553): x f32 [batch, C, H, W, D] -> zero pad H, W to even at
 * the bottom / right -> 2x2 gather with feature order (h w D) -> LayerNorm(4D) with affine gamma/beta
 * -> bf16 [batch*C*ceil(H/2)*ceil(W/2), 4D], the A operand of `reduction` (ab_gemm_bf16). */
int ab_patch_merge_ln(const float* x, const float* gamma, const float* beta, void* out_bf16, int32_t batch,
                      int32_t c, int32_t h, int32_t w, int32_t d, float eps, void* stream);

/* PatchSplitting3D middle (swin3d.py:585-611): y bf16 [batch*C*H*W, 2D] (output of lin1) -> view
 * (.., 2, 2, D/2) pixel shuffle to (2H, 2W) -> crop the merge padding (crop_h, crop_w in {0,1}, removed at
 * the bottom / right) -> LayerNorm(D/2) affine -> bf16 [batch*C*(2H-crop_h)*(2W-crop_w), D/2], the A
 * operand of lin2.  `d` is the layer's input dimension D. */
int ab_patch_split_ln(const void* y_bf16, const float* gamma, const float* beta, void* out_bf16, int32_t batch,
                      int32_t c, int32_t h, int32_t w, int32_t d, int32_t crop_h, int32_t crop_w, float eps,
                      void* stream);

/* Perceiver cross-attention core (perceiver.py:148-151) for location-independent queries:
 * q f32 [lq, D] (= to_q(latents), computed once), kv bf16 [lk*nloc, ld_kv] with row = ck*nloc + loc and
 * columns [k | v]; out bf16 [lq*nloc, ld_out], row = cq*nloc + loc.  softmax(q k^T / sqrt(head_dim)) v
 * per (location, head); head_dim 32 or 64. */
int ab_perceiver_attention(const float* q, const void* kv_bf16, void* out_bf16, int64_t nloc, int32_t lq,
                           int32_t lk, int32_t num_heads, int32_t head_dim, int32_t ld_kv, int32_t ld_out,
                           int32_t dtype /* AB_DT_* of kv and out */, void* stream);

/* y f32 [rows, n] = silu_out?( silu_in?(x f32 [rows, k]) W^T + bias ), W f32 [n, k]: the handful of
 * location-independent vectors (time MLP swin3d.py:805-809,914; adaLN modulation film.py:27-28; level,
 * lead-time and absolute-time embeddings encoder.py:323-325,352-363, decoder.py:220-223). */
int ab_linear_small_f32(const float* x, const float* w, const float* bias, float* y, int32_t rows, int32_t n,
                        int32_t k, int32_t silu_in, int32_t silu_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Batch <-> token matrix.  Field descriptors are HOST arrays (copied into the launch).
 * ---------------------------------------------------------------------------------------------- */
#define AB_MAX_FIELDS 64

enum {
  AB_IN_PLAIN = 0,
  AB_IN_CLAMP_MIN0 = 1,
  AB_IN_CLAMP_LOG_COMBINE = 2,
  /* AuroraWave._pre_encoder_hook (aurora.py:874-892), applied to the NORMALISED value z: */
  AB_IN_NAN_TO_ZERO = 3, /* z.nan_to_num(0)                              (value channel of a density variable) */
  AB_IN_DENSITY = 4,     /* (~isnan(z)).float()                          (`<name>_density`) */
  AB_IN_SIN_DEG = 5,     /* sin(deg2rad(z)).nan_to_num(0)                (`<name>_sin`) */
  AB_IN_COS_DEG = 6      /* cos(deg2rad(z)).nan_to_num(0)                (`<name>_cos`) */
};

typedef struct AbFieldIn {
  const float* ptr;   /* (T, H, W) planes of one variable (one batch element, one level); NULL = constant */
  int64_t stride_t;   /* elements between history steps (0 for static variables) */
  float loc, scale;   /* normalisation (x - loc) / scale   (batch.py:94-116, normalisation.py:34-70) */
  float const_value;  /* normalised value when ptr == NULL (dynamic time-of-day style variables) */
  int32_t transform;  /* AB_IN_* : positive clamp (aurora.py:302-317) / AirPollution combiner (:733-742) /
                         AuroraWave density + angle channels (:874-892) */
  float w0, w1, wb;   /* combiner Linear(2,1) weights and bias */
} AbFieldIn;

/* out bf16 [ (H/p)*(W/p), ldk ] with column ((v*t_hist + t)*p + p1)*p + p2 = transform(field v at history t,
 * pixel (hp*p + p1, wp*p + p2)); columns >= nfields*t_hist*p*p are left untouched (keep them zero).
 * Replaces Batch.normalise + torch.stack (encoder.py:213-215) + conv3d im2col (patchembed.py:100-112). */
int ab_patchify(const AbFieldIn* fields, int32_t nfields, int32_t t_hist, int32_t h, int32_t w, int32_t p,
                void* out_bf16, int32_t ldk, int32_t out_dtype /* AB_DT_* */, void* stream);

typedef struct AbFieldOut {
  float* ptr;         /* (H, W) output plane, physical units */
  const float* prev;  /* previous state plane (row pitch W), physical units; needed when mod_col >= 0 */
  float loc, scale;   /* un-normalisation y * scale + loc (batch.py:118-140) */
  int32_t col;        /* first of the p*p head columns of this variable in y */
  int32_t mod_col;    /* first column of its modulation head (aurora.py:767-775) or -1 */
  int32_t clamp_min0; /* positive-variable clamp (aurora.py:367-388) */
  int32_t clamp_max1; /* AirPollution SO2 >= 850 hPa clamp (aurora.py:787-794) */
  /* AuroraWave._post_decoder_hook (aurora.py:894-920); all in normalised units, before y * scale + loc: */
  int32_t cos_col;    /* >= 0: `col` holds the sine head, this the cosine head; value = rad2deg(atan2(s, c)) mod 360 */
  int32_t dens_col;   /* >= 0: density-logit head; value *= m, NaN where sigmoid(logit) * m < 0.5, m = mask > mask_min */
  const float* mask;  /* (H, W) plane of the `wmb` static variable, physical units; needed when dens_col >= 0 */
  float mask_min;     /* physical-unit threshold equivalent to "normalised wmb > 0" (= its location) */
} AbFieldOut;

/* y f32 [ (H/p)*(W/p), ldy ] (head GEMM output, column col + p1*p + p2) -> planes.  Replaces torch.stack +
 * unpatchify (decoder.py:214-217,250-263; util.py:18-41), the post-decoder hooks and Batch.unnormalise. */
int ab_unpatchify(const AbFieldOut* fields, int32_t nfields, const float* y, int32_t ldy, int32_t h, int32_t w,
                  int32_t p, void* stream);

typedef struct AbOp {
  int32_t kind; /* AB_OP_* */
  int32_t reserved_;
  union {
    AbGemm gemm;
    AbSwinBlock block;
    AbLnModResidual ln;
    AbPatchMergeLn merge;
    AbPatchSplitLn split;
  } u;
} AbOp;

int ab_run_ops(const AbOp* ops, int32_t n_ops, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Tropical-cyclone tracking on device-resident predictions (the reference's aurora/tracker.py:61-104,
 * 185-196, 262-282): ONE launch evaluates
 * a list of boxes, one CTA per box, and writes a few bytes per box; the scalar decisions stay with the caller.  A box
 * is the cross product of a row-index list and a column-index list into one field plane (lists, because the
 * reference's longitude selection wraps around and concatenates two ranges, :36-47).
 *
 *   AB_TRACK_MINIMA   masks[mask_off ..] = uint8 [n_rows, n_cols] row-major: the local minima of the box after
 *                     scipy.ndimage.gaussian_filter(box, sigma=1) (radius 4, float64 accumulation, rounded to f32 per
 *                     axis) and an 8 x 8 minimum filter, both with mode "reflect"; border rows / columns cleared.
 *                     counts[i] = number of minima.
 *   AB_TRACK_MAX      values[i] = max of the box                 (the land test `lsm_box.max() < 0.5`)
 *   AB_TRACK_MIN      values[i] = min of the box                 (minimum msl of the crop)
 *   AB_TRACK_WINDMAX  values[i] = max of sqrt(u*u + v*v), u = plane, v = plane2, each operation rounded as numpy
 *                     float32 does
 * Reductions propagate NaN like numpy.  The index lists are DEVICE int32 memory (`index`); every entry is checked
 * against the plane's extent in the kernel, and a box with an entry outside it gets counts[i] = -1 and values[i] = NaN.
 * `boxes` is a HOST array; `box_bytes` must be sizeof(AbTrackBox).  1 <= n_rows, n_cols <= AB_TRACK_MAX_SIDE and
 * n_boxes <= AB_TRACK_MAX_BOXES (the descriptors travel as kernel parameters); larger boxes are AB_ERR_UNSUPPORTED.
 * ---------------------------------------------------------------------------------------------- */
enum { AB_TRACK_MINIMA = 0, AB_TRACK_MAX = 1, AB_TRACK_MIN = 2, AB_TRACK_WINDMAX = 3 };
#define AB_TRACK_MAX_SIDE 101 /* delta 5 at 0.1 degrees, the finest grid of the shipped models */
#define AB_TRACK_MAX_BOXES 32

typedef struct AbTrackBox {
  const float* plane;  /* f32 [h, ld] */
  const float* plane2; /* AB_TRACK_WINDMAX: the v plane, same layout as `plane`; NULL otherwise */
  int32_t h, w, ld;    /* extent of the plane and elements between its rows */
  int32_t op;          /* AB_TRACK_* */
  int32_t rows_off, n_rows; /* row indices: index[rows_off .. rows_off + n_rows) */
  int32_t cols_off, n_cols; /* column indices: index[cols_off .. cols_off + n_cols) */
  int64_t mask_off;    /* AB_TRACK_MINIMA: byte offset of the box's mask in `masks` */
} AbTrackBox;

int ab_track_boxes(const AbTrackBox* boxes, int32_t n_boxes, size_t box_bytes, const int32_t* index, float* values,
                   int32_t* counts, uint8_t* masks, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Latitude-weighted scores of device-resident predictions against a truth (and a climatology): the sums behind
 * RMSE, bias, MAE and the uncentred anomaly correlation, for every level plane of every field, in one call.  Not a
 * reference function: the reference's notebooks copy each prediction to the host and score it in numpy.
 *
 * One AbScoreField per variable (and batch member): `levels` planes of h x w float32 values in each of pred, truth and
 * clim (clim may be NULL), row pitch ld_*, `*_level_stride` elements between planes.  Planes are numbered field by
 * field, level by level.  For plane p, with w_r = row_weights[r] (double [h] of the largest h, DEVICE memory) and the
 * point valid when pred, truth and (if given) clim are all not NaN, sums[p][0..7] =
 *   W = sum w_r,  sum w_r d,  sum w_r d^2,  sum w_r |d|,  sum w_r af ao,  sum w_r af^2,  sum w_r ao^2,  count,
 * over the valid points, d = double(pred) - double(truth), af = double(pred) - double(clim),
 * ao = double(truth) - double(clim); the last three are 0 without clim.  +-inf is not skipped.  Every element is
 * read once with float64 arithmetic; rows are split into a fixed (plane, row-chunk) partition whose partial sums go to
 * `workspace` and are added in a fixed order by a second launch, so repeated calls give bit-identical sums (no
 * atomics).  `fields` is a HOST array copied into the launch; `field_bytes` must be sizeof(AbScoreField);
 * 1 <= n_fields <= AB_SCORE_MAX_FIELDS; h, w, levels >= 1, ld_* >= w; 16-byte loads where every pointer, pitch and
 * level stride of a field allow, scalar loads otherwise.  `sums` is double [total planes][8], DEVICE memory.
 * ---------------------------------------------------------------------------------------------- */
#define AB_SCORE_MAX_FIELDS 64
#define AB_SCORE_SUMS 8

typedef struct AbScoreField {
  const float* pred;  /* f32 [levels][h, ld_pred] */
  const float* truth; /* f32 [levels][h, ld_truth] */
  const float* clim;  /* f32 [levels][h, ld_clim] or NULL */
  int64_t pred_level_stride, truth_level_stride, clim_level_stride; /* elements between consecutive levels */
  int32_t h, w;
  int32_t ld_pred, ld_truth, ld_clim;
  int32_t levels;
} AbScoreField;

/* Workspace `ab_score_fields` needs for these fields (validates them like it does).  Host only. */
int ab_score_workspace_bytes(const AbScoreField* fields, int32_t n_fields, size_t field_bytes, size_t* bytes);
int ab_score_fields(const AbScoreField* fields, int32_t n_fields, size_t field_bytes, const double* row_weights,
                    double* sums, void* workspace, size_t workspace_bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Latitude-weighted scores of a device-resident ensemble against a truth (and a climatology): the sums behind the
 * ensemble-mean RMSE and bias, the spread, the fair CRPS and the ensemble-mean ACC, for every level plane of every
 * field, in one call.  Not a reference function.
 *
 * One AbEnsembleField per variable: n_members (2 <= M <= AB_ENS_MAX_MEMBERS) member pointers that share one row pitch
 * ld_member and one level stride, a truth and a clim (may be NULL), each `levels` planes of h x w float32 values.
 * Planes are numbered field by field, level by level.  For plane p, with w_r = row_weights[r] (double [h] of the
 * largest h, DEVICE memory), a point valid when the truth, every member and (if given) clim are all not NaN, x_k the
 * member values, xm their mean, s2 their unbiased variance (all in double), y = truth and c = clim,
 * sums[p][0..9] =
 *   W = sum w_r,  sum w_r (xm - y),  sum w_r (xm - y)^2,  sum w_r s2,  sum w_r (1/M) sum_k |x_k - y|,
 *   sum w_r (1/(M(M-1))) sum_{k != l} |x_k - x_l|,  sum w_r af ao,  sum w_r af^2,  sum w_r ao^2,  count,
 * over the valid points, af = xm - c, ao = y - c; sums 6..8 are 0 without clim.  +-inf is not skipped.  Each point's
 * member values are sorted (a bitonic network over 8, 16, 32 or 64 values, the smallest that holds the largest M of
 * the call) and every per-point quantity is formed in that order, so the sums do not depend on the order of the
 * members, bit for bit.  Rows are split into a fixed (plane, row-chunk) partition whose partial sums go to
 * `workspace` and are added in a fixed order by a second launch, so repeated calls give bit-identical sums (no
 * atomics).  `fields` is a HOST array copied into the launch; `field_bytes` must be sizeof(AbEnsembleField);
 * 0 <= n_fields <= AB_ENS_MAX_FIELDS (0 is a no-op); h, w, levels >= 1, ld_* >= w, level strides >= 0; 16-byte loads
 * where every pointer, pitch, level stride and the width of a field allow, scalar loads otherwise.  `sums` is
 * double [total planes][AB_ENS_SUMS], DEVICE memory.
 * ---------------------------------------------------------------------------------------------- */
#define AB_ENS_MAX_MEMBERS 64
#define AB_ENS_MAX_FIELDS 16 /* the 9 variables of the 1.3 B model in one call; the launch parameter is ~9.6 KB */
#define AB_ENS_SUMS 10

typedef struct AbEnsembleField {
  const float* members[AB_ENS_MAX_MEMBERS]; /* the first n_members: f32 [levels][h, ld_member] each */
  const float* truth;                       /* f32 [levels][h, ld_truth] */
  const float* clim;                        /* f32 [levels][h, ld_clim] or NULL */
  int64_t member_level_stride, truth_level_stride, clim_level_stride; /* elements between consecutive levels */
  int32_t n_members;
  int32_t h, w;
  int32_t ld_member, ld_truth, ld_clim;
  int32_t levels;
} AbEnsembleField;

/* Workspace `ab_ensemble_score_fields` needs for these fields (validates them like it does).  Host only. */
int ab_ensemble_score_workspace_bytes(const AbEnsembleField* fields, int32_t n_fields, size_t field_bytes,
                                      size_t* bytes);
int ab_ensemble_score_fields(const AbEnsembleField* fields, int32_t n_fields, size_t field_bytes,
                             const double* row_weights, double* sums, void* workspace, size_t workspace_bytes,
                             void* stream);

/* ------------------------------------------------------------------------------------------------
 * Latitude-band zonal power spectra of device-resident fields: for every level plane of every field and every band,
 * the latitude-weighted mean over the band's rows of each row's one-sided variance spectrum, in one call.  Not a
 * reference function: the reference's notebooks copy each prediction to the host and use numpy.fft.
 *
 * One AbSpectrumField per variable (and batch member): `levels` planes of h x w float32 values, row pitch ld,
 * `level_stride` elements between planes; every field of a call has the same h and w.  Planes are numbered field by
 * field, level by level.  Band b is the rows [band_rows[2b], band_rows[2b + 1]) (a HOST array).  For a row x_0..x_{N-1}
 * (N = w), X_k = sum_n x_n e^{-2 pi i k n / N} in double and P(k) = c_k |X_k|^2 / N^2 for k = 0..N/2, c_k = 1 for
 * k = 0 and (N even) k = N/2, else 2, so that sum_k P(k) = (1/N) sum_n x_n^2.  A row counts when all its N values are
 * finite.  With w_r = row_weights[r] (double [h], DEVICE memory), out[p][b][0..N/2+2] =
 *   sum w_r,  rows,  sum w_r P_r(0),  ...,  sum w_r P_r(N/2)
 * over the counted rows of band b of plane p.  Each row is staged in shared memory (cp.async.bulk where the row
 * address and 4 w bytes are 16-byte multiples, cp.async otherwise) and transformed two rows at a time as one complex
 * mixed-radix (4 / 2 / 3 / 5) FFT in double.  Rows are split into a fixed (plane, band, row-chunk) partition whose
 * partial sums go to `workspace` and are added in a fixed order by a second launch, so repeated calls give
 * bit-identical sums (no atomics).  `fields` is a HOST array copied into the launch; `field_bytes` must be
 * sizeof(AbSpectrumField); 0 <= n_fields <= AB_SPEC_MAX_FIELDS (0 is a no-op); 1 <= n_bands <= AB_SPEC_MAX_BANDS;
 * 0 <= band_rows[2b] <= band_rows[2b + 1] <= h; h, levels >= 1; 1 <= w <= AB_SPEC_MAX_WIDTH with no prime factor
 * above 5; ld >= w, level_stride >= 0.  `out` is double [total planes][n_bands][w/2 + 3], DEVICE memory.
 * ---------------------------------------------------------------------------------------------- */
#define AB_SPEC_MAX_FIELDS 64 /* the 9 variables of the 1.3 B model for up to 7 members in one call */
#define AB_SPEC_MAX_BANDS 8
#define AB_SPEC_MAX_WIDTH 4096

typedef struct AbSpectrumField {
  const float* x;       /* f32 [levels][h, ld] */
  int64_t level_stride; /* elements between consecutive levels */
  int32_t h, w, ld;
  int32_t levels;
} AbSpectrumField;

/* Workspace `ab_zonal_spectra` needs for these fields and bands (validates them like it does).  Host only. */
int ab_zonal_spectra_workspace_bytes(const AbSpectrumField* fields, int32_t n_fields, size_t field_bytes,
                                     const int32_t* band_rows, int32_t n_bands, size_t* bytes);
int ab_zonal_spectra(const AbSpectrumField* fields, int32_t n_fields, size_t field_bytes, const int32_t* band_rows,
                     int32_t n_bands, const double* row_weights, double* out, void* workspace, size_t workspace_bytes,
                     void* stream);

/* sizeof() of the descriptor structs as this library was compiled (binding authors: compare with your mirror).
 * which: 0 AbGemm, 1 AbWindowAttention, 2 AbLnModResidual, 3 AbFieldIn, 4 AbFieldOut, 5 AbHaloPush, 6 AbSwinBlock,
 * 7 AbGemmLn, 8 AbPatchMergeLn, 9 AbPatchSplitLn, 10 AbOp; -1 for an unknown index.  Host only. */
int ab_struct_size(int32_t which);

#ifdef __cplusplus
}
#endif

#endif /* AURORA_B200_H_ */
