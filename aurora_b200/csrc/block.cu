// Whole-block entry point: one call runs a complete Swin3DTransformerBlock (aurora/model/swin3d.py:440-509) on the
// flat token stream — what the reference does in ~40 ATen / cuBLAS / SDPA calls per block:
//
//   qkv   = x_b16 · Wqkv^T + b                      (wgmma GEMM; LoRA already merged into Wqkv, lora.py:104-129)
//   [latitude slab: push K | V halo rows to the neighbours, wait for theirs            csrc/halo.cu]
//   att   = shifted-window attention(qkv)           (roll / pad / partition / mask / SDPA / reverse / crop / un-roll)
//   y     = att · Wproj^T + b
//   x     = x + LN(y) * scale1 + shift1             (AdaptiveLayerNorm, film.py:48-49; fp32 stream + 16-bit copy)
//   h     = GELU_erf(x_b16 · Wfc1^T + b)
//   y     = h · Wfc2^T + b
//   x     = x + LN(y) * scale2 + shift2
// With `fuse_ln` and D = 512 / 1024 each "projection, then x = x + LN(y) ..." pair is ONE kernel (csrc/gemm_ln.cu):
// the adaLN + residual runs in the projection's epilogue and y never reaches HBM.
//
// It only sequences the kernels of this library on the caller's stream (8 - 10 launches); the caller (PyTorch) owns
// every buffer, the workspace included (ab_swin_block_workspace_bytes).
#include "common.h"

namespace {

inline size_t align256(size_t x) { return (x + 255) & ~static_cast<size_t>(255); }

struct BlockWs {
  size_t qkv, att, y, hid, total;
};

BlockWs layout(long long tokens, int dim, int hidden) {
  BlockWs w;
  size_t off = 0;
  w.qkv = off;
  off += align256(static_cast<size_t>(tokens) * 3 * dim * 2);
  w.att = off;
  off += align256(static_cast<size_t>(tokens) * dim * 2);
  w.y = off;
  off += align256(static_cast<size_t>(tokens) * dim * 2);
  w.hid = off;
  off += align256(static_cast<size_t>(tokens) * hidden * 2);
  w.total = off;
  return w;
}

}  // namespace

extern "C" int ab_swin_block_workspace_bytes(int64_t tokens, int32_t dim, int32_t hidden, size_t* bytes) {
  using namespace ab;
  AB_CHECK_ARG(bytes != nullptr && tokens > 0 && dim > 0 && hidden > 0, "ab_swin_block_workspace_bytes: bad argument");
  *bytes = layout(tokens, dim, hidden).total;
  return AB_OK;
}

extern "C" int ab_swin_block(const AbSwinBlock* b, void* stream) {
  using namespace ab;
  AB_CHECK_ARG(b != nullptr, "ab_swin_block: null descriptor");
  AB_CHECK_ARG(b->x_f32 && b->x_b16 && b->workspace && b->w_qkv && b->w_proj && b->w_fc1 && b->w_fc2 && b->b_qkv &&
                   b->b_proj && b->b_fc1 && b->b_fc2 && b->scale1 && b->shift1 && b->scale2 && b->shift2,
               "ab_swin_block: null pointer in the descriptor");
  AB_CHECK_ARG(b->dim > 0 && b->hidden > 0 && b->num_heads > 0 && b->dim == b->num_heads * 64,
               "ab_swin_block: dim (%d) must be num_heads (%d) x 64", b->dim, b->num_heads);
  AB_CHECK_ARG((reinterpret_cast<uintptr_t>(b->workspace) & 255u) == 0, "ab_swin_block: workspace must be 256-byte aligned");
  const bool slab = b->slab_h_rows > 0;
  const long long tokens = slab ? static_cast<long long>(b->res[0]) * b->slab_h_rows * b->res[2]
                                : static_cast<long long>(b->res[0]) * b->res[1] * b->res[2];
  AB_CHECK_ARG(tokens > 0 && tokens < (1ll << 31), "ab_swin_block: bad token count");
  const BlockWs ws = layout(tokens, b->dim, b->hidden);
  uint8_t* base = reinterpret_cast<uint8_t*>(b->workspace);
  void* qkv = base + ws.qkv;
  void* att = base + ws.att;
  void* y = base + ws.y;
  void* hid = base + ws.hid;
  const int m = static_cast<int>(tokens), d = b->dim;
  int rc;

  AbGemm g = {};
  g.in_dtype = AB_DT_BF16;
  g.out_dtype = AB_DT_BF16;
  g.m = m;
  // qkv projection
  g.a = b->x_b16, g.w = b->w_qkv, g.bias = b->b_qkv, g.out_bf16 = qkv;
  g.n = 3 * d, g.k = d, g.lda = d, g.ldw = d, g.ld_bf16 = 3 * d;
  // fused compute + exchange: the projection's epilogue stores the boundary K | V rows into the neighbours' memory
  const bool slab_push = b->slab_h_rows > 0 && b->halo_push != nullptr;
  const bool fused_push = slab_push && b->fuse_push != 0 && (b->halo_push->rows_to_above + b->halo_push->rows_to_below) > 0 &&
                          2 * b->halo_push->c <= 8;
  if (fused_push) g.peer_push = b->halo_push;
  if ((rc = ab_gemm_bf16(&g, stream)) != AB_OK) return rc;
  g.peer_push = nullptr;

  AbWindowAttention a = {};
  a.qkv = qkv, a.pad_qkv = b->pad_qkv, a.out = att;
  a.batch = 1, a.num_heads = b->num_heads, a.head_dim = 64, a.warped = 1;
  for (int i = 0; i < 3; ++i) a.res[i] = b->res[i], a.window[i] = b->window[i], a.shift[i] = b->shift[i];
  if (slab) {
    if (b->halo_push != nullptr) {  // peer transport: my boundary K | V rows go to the neighbours ...
      if (!fused_push) {            // ... by the copy kernel, unless the projection above has already sent them
        AbHaloPush hp = *b->halo_push;
        hp.local = qkv;
        if ((rc = ab_halo_push(&hp, stream)) != AB_OK) return rc;
      }
      a.halo_ctrl = b->halo_push->ctrl;  // the attention kernel waits for the neighbours' rows itself, interior windows first
    }
    a.slab_h_begin = b->slab_h_begin, a.slab_h_rows = b->slab_h_rows, a.slab_halo = b->halo_rows;
    a.halo_kv = b->halo_kv;
  }
  if ((rc = ab_window_attention(&a, stream)) != AB_OK) return rc;

  // adaLN + residual fused into the epilogue of the projection / fc2 where a cluster can own whole rows (csrc/gemm_ln.cu)
  const bool fuse = b->fuse_ln != 0 && ab_gemm_ln_supported(d) != 0;
  AbGemmLn gl = {};
  gl.in_dtype = AB_DT_BF16, gl.out_dtype = AB_DT_BF16, gl.eps = b->eps;
  gl.m = m, gl.n = d, gl.ldr = d, gl.ld_f32 = d, gl.ld_16 = d;
  gl.residual = b->x_f32, gl.out_f32 = b->x_f32, gl.out_16 = b->x_b16;

  // output projection + adaLN 1 + residual
  if (fuse) {
    gl.a = att, gl.w = b->w_proj, gl.bias = b->b_proj, gl.scale = b->scale1, gl.shift = b->shift1;
    gl.k = d, gl.lda = d, gl.ldw = d;
    if ((rc = ab_gemm_ln_residual(&gl, stream)) != AB_OK) return rc;
  }
  g.a = att, g.w = b->w_proj, g.bias = b->b_proj, g.out_bf16 = y;
  g.n = d, g.k = d, g.lda = d, g.ldw = d, g.ld_bf16 = d;
  if (!fuse && (rc = ab_gemm_bf16(&g, stream)) != AB_OK) return rc;
  AbLnModResidual ln = {};
  ln.y = y, ln.scale = b->scale1, ln.shift = b->shift1, ln.residual = b->x_f32, ln.out_f32 = b->x_f32, ln.out_bf16 = b->x_b16;
  ln.rows = m, ln.dim = d, ln.ld_y = d, ln.ld_res = d, ln.ld_f32 = d, ln.ld_bf16 = d, ln.eps = b->eps;
  ln.in_dtype = AB_DT_BF16, ln.out_dtype = AB_DT_BF16;
  if (!fuse && (rc = ab_ln_mod_residual(&ln, stream)) != AB_OK) return rc;

  // MLP + adaLN 2 + residual
  g.a = b->x_b16, g.w = b->w_fc1, g.bias = b->b_fc1, g.out_bf16 = hid, g.act = AB_ACT_GELU_ERF;
  g.n = b->hidden, g.k = d, g.lda = d, g.ldw = d, g.ld_bf16 = b->hidden;
  if ((rc = ab_gemm_bf16(&g, stream)) != AB_OK) return rc;
  if (fuse) {
    gl.a = hid, gl.w = b->w_fc2, gl.bias = b->b_fc2, gl.scale = b->scale2, gl.shift = b->shift2;
    gl.k = b->hidden, gl.lda = b->hidden, gl.ldw = b->hidden;
    if (b->out_b16 != nullptr) gl.out_16 = b->out_b16, gl.ld_16 = b->ld_out_b16, gl.out_dtype = b->out_b16_dtype;
    return ab_gemm_ln_residual(&gl, stream);
  }
  g.a = hid, g.w = b->w_fc2, g.bias = b->b_fc2, g.out_bf16 = y, g.act = AB_ACT_NONE;
  g.n = d, g.k = b->hidden, g.lda = b->hidden, g.ldw = b->hidden, g.ld_bf16 = d;
  if ((rc = ab_gemm_bf16(&g, stream)) != AB_OK) return rc;
  ln.scale = b->scale2, ln.shift = b->shift2;
  if (b->out_b16 != nullptr) {  // the 16-bit copy of the block output goes elsewhere (e.g. into the skip concatenation)
    ln.out_bf16 = b->out_b16, ln.ld_bf16 = b->ld_out_b16, ln.out_dtype = b->out_b16_dtype;
  }
  return ab_ln_mod_residual(&ln, stream);
}

extern "C" int ab_run_ops(const AbOp* ops, int32_t n_ops, void* stream) {
  using namespace ab;
  AB_CHECK_ARG(ops != nullptr && n_ops >= 0, "ab_run_ops: null list");
  for (int i = 0; i < n_ops; ++i) {
    const AbOp& op = ops[i];
    int rc;
    switch (op.kind) {
      case AB_OP_GEMM:
        rc = ab_gemm_bf16(&op.u.gemm, stream);
        break;
      case AB_OP_SWIN_BLOCK:
        rc = ab_swin_block(&op.u.block, stream);
        break;
      case AB_OP_LN_MOD_RESIDUAL:
        rc = ab_ln_mod_residual(&op.u.ln, stream);
        break;
      case AB_OP_PATCH_MERGE_LN: {
        const AbPatchMergeLn& m = op.u.merge;
        rc = ab_patch_merge_ln(m.x, m.gamma, m.beta, m.out_bf16, m.batch, m.c, m.h, m.w, m.d, m.eps, stream);
        break;
      }
      case AB_OP_PATCH_SPLIT_LN: {
        const AbPatchSplitLn& sp = op.u.split;
        rc = ab_patch_split_ln(sp.y_bf16, sp.gamma, sp.beta, sp.out_bf16, sp.batch, sp.c, sp.h, sp.w, sp.d, sp.crop_h,
                               sp.crop_w, sp.eps, stream);
        break;
      }
      default:
        set_error("ab_run_ops: unknown operation kind %d at index %d", op.kind, i);
        return AB_ERR_INVALID_ARGUMENT;
    }
    if (rc != AB_OK) return rc;  // ab_last_error() describes the failing operation
  }
  return AB_OK;
}

extern "C" int ab_struct_size(int32_t which) {
  switch (which) {
    case 0: return static_cast<int>(sizeof(AbGemm));
    case 1: return static_cast<int>(sizeof(AbWindowAttention));
    case 2: return static_cast<int>(sizeof(AbLnModResidual));
    case 3: return static_cast<int>(sizeof(AbFieldIn));
    case 4: return static_cast<int>(sizeof(AbFieldOut));
    case 5: return static_cast<int>(sizeof(AbHaloPush));
    case 6: return static_cast<int>(sizeof(AbSwinBlock));
    case 7: return static_cast<int>(sizeof(AbGemmLn));
    case 8: return static_cast<int>(sizeof(AbPatchMergeLn));
    case 9: return static_cast<int>(sizeof(AbPatchSplitLn));
    case 10: return static_cast<int>(sizeof(AbOp));
    default: return -1;
  }
}
