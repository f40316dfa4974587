/* omnidata_b200 — C ABI of the H100-native (sm_90a) DPT-Hybrid-384 hot path.
 *
 * This header is the drop-in boundary (SURVEY.md §8b).  The reference (EPFL-VILAB/omnidata) is pure
 * Python/PyTorch on this path and has no FFI of its own; every entry point below replaces a chain
 * of torch library calls made by a reference function, cited as `file:line` under
 * omnidata_tools/torch/ (M/ = modules/midas/, L/ = losses/).  timm 0.4.12 (pinned by
 * requirements.txt:15, called at M/vit.py:483) is not vendored in the reference; its arithmetic
 * is cited as "timm <symbol>".
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless the name says host; no torch types cross this ABI;
 *   - activations are channels-last (NHWC / token-major) bf16 unless stated; strides are in
 *     ELEMENTS, the channel stride is always 1;
 *   - an `int32_t dtype` (or x_dtype / y_dtype) parameter is an odb_dtype naming the storage type of the
 *     activation tensors of that call (bf16 in production, fp32 in the correctness mode);
 *   - every function only enqueues work on `stream` (a cudaStream_t passed as void*); nothing
 *     allocates, synchronises or touches the host heap — safe under CUDA-graph capture;
 *   - return value: 0 on success, a negative odb_status otherwise; odb_last_error() returns a
 *     thread-local message.  There is NO CPU fallback: without a CUDA device every compute entry
 *     point fails with ODB_ERR_CUDA.
 */
#ifndef OMNIDATA_B200_H_
#define OMNIDATA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ODB_ABI_VERSION 4

typedef enum odb_status {
  ODB_OK = 0,
  ODB_ERR_INVALID = -1, /* bad argument / unsupported shape */
  ODB_ERR_CUDA = -2,    /* CUDA runtime or driver error (message has the detail) */
  ODB_ERR_UNSUPPORTED = -3
} odb_status;

typedef enum odb_act { ODB_ACT_NONE = 0, ODB_ACT_RELU = 1, ODB_ACT_GELU = 2 } odb_act;

/* Storage type of an activation tensor.  bf16 is the production format; fp32 carries the ViT residual stream
 * (the reference adds every block's output to an fp32 stream: timm Block.forward `x = x + ...`) and every
 * activation of the fp32 correctness mode (SURVEY.md 8c: the reference itself is fp32-only).  e4m3 (FP8, 1 byte,
 * OCP E4M3FN: finite range +-448) is the operand type of the fp8 inference mode's ViT linear layers, always paired with
 * fp32 scale vectors (odb_conv_gemm_scaled, odb_layernorm_e4m3, odb_rowquant_e4m3). */
typedef enum odb_dtype { ODB_DTYPE_BF16 = 0, ODB_DTYPE_F32 = 1, ODB_DTYPE_E4M3 = 2 } odb_dtype;

/* A strided channels-last view [b][h][w][c] (bf16 storage unless the owning descriptor says fp32; strides in
 * elements of the storage type). */
typedef struct odb_view {
  const void* ptr;
  int32_t c, w, h, b;
  int64_t sx, sy, sb; /* element strides of w, h, b */
} odb_view;

#define ODB_MAX_VIEWS 4
#define ODB_MAX_TAPS 9

/* Implicit-GEMM convolution / linear layer on Hopper tensor cores (wgmma):
 *
 *   out[b,y,x,n] = epilogue( sum_{t<num_taps} sum_{c<C} view[tap_view[t]][b, y+tap_dy[t], x+tap_dx[t], c]
 *                                                     * weight[n][t*C + c] )
 *
 * Reads outside a view are zero (TMA out-of-bounds fill) — this is the convolution padding.
 * A stride-2 convolution is expressed with up to four parity-plane views (doubled strides).
 * A linear layer is the degenerate case num_taps = 1, h = b = 1, w = rows.
 *
 * epilogue(v) = residual + act(v + bias)        (each term optional), stored as bf16 to `out`
 *               and, if out2.ptr != NULL, relu(.) of the same value to `out2`.
 *
 * Replaces, depending on the call site: nn.Linear in timm Attention/Mlp (loop M/vit.py:150-151),
 * timm HybridEmbed.proj (M/vit.py:133), ProjectReadout.project (M/vit.py:36-47),
 * act_postprocess convs (M/vit.py:431-462), scratch.layerN_rn (M/blocks.py:49-75, used
 * M/dpt_depth.py:73-76), ResidualConvUnit_custom.conv1/conv2 (M/blocks.py:263-286),
 * FeatureFusionBlock_custom.out_conv (M/blocks.py:339), output_conv[0] (M/dpt_depth.py:91),
 * timm ResNetV2 StdConv2dSame layers.
 */
typedef struct odb_conv_gemm_desc {
  int32_t num_views;
  odb_view views[ODB_MAX_VIEWS]; /* all views share c = C (multiple of 8; K blocks of 64) */
  int32_t num_taps;
  int8_t tap_view[ODB_MAX_TAPS];
  int8_t tap_dx[ODB_MAX_TAPS];
  int8_t tap_dy[ODB_MAX_TAPS];
  const void* weight; /* bf16 [n][num_taps * C], K contiguous */
  int32_t n;          /* output channels */
  odb_view out;       /* c = n; w,h,b = output extent */
  odb_view out2;      /* optional relu copy (ptr may be NULL) */
  const float* bias;  /* fp32 [n] or NULL */
  int64_t bias_sb;    /* 0, or n for a per-image bias [b][n] (ProjectReadout cls term) */
  odb_view residual;  /* optional bf16 residual, same extent as out (ptr may be NULL); sb may be 0 */
  int32_t act;        /* odb_act */
  int32_t tile_w, tile_h; /* spatial tile of the 128-row MMA tile, tile_w*tile_h <= 128; 0 = auto */
  int32_t block_n;        /* N tile: 256, 128, 64 (32 with the head tail); 0 = auto */
  int32_t cta_pair;       /* CTA pair: a 2-CTA cluster takes two adjacent 128-row tiles and shares the weight tile by TMA multicast
                           * (block_n 256, or 128 without halo; no head tail): 1 = on, 0 / -1 = off */
  int32_t halo;           /* 3x3 stride-1 pad-1 convs: load one halo tile per K block and address the nine
                           * taps inside it (3x less input traffic): 0 = auto (currently off: the deeper per-tap ring measured
                           * faster on every layer of this network), 1 = on, -1 = off */
  /* Fused DPT head tail (M/dpt_depth.py:93-97): only with n == 32.  When head_out != NULL the
   * 32-channel result relu(v + bias) is not stored; instead
   *   head_out[b][k][y][x] = relu?(head_b[k] + sum_j head_w[k][j] * relu(v_j + bias_j))  (fp32, NCHW) */
  const float* head_w; /* fp32 [head_c][32] */
  const float* head_b; /* fp32 [head_c] */
  int32_t head_c;
  int32_t head_relu;
  float* head_out;
  /* Fused GroupNorm statistics (timm GroupNormAct after every StdConv2dSame): when gn_partial != NULL
   * each epilogue warp also writes, for the rows it owns, the per-group (sum, sum of squares)
   * of its 32 rows to  gn_partial[b][ty*tiles_x+tx][quadrant 0..3][group][2]  (fp32, every entry is
   * written exactly once: no atomics, deterministic).  The sums are taken over the UNROUNDED fp32 accumulators
   * (timm GroupNormAct normalises the fp32 conv output), not over the stored bf16 values.  odb_groupnorm_finalize reduces them. */
  float* gn_partial;
  int32_t gn_groups;
  /* Epilogue code path: 0 = auto (a specialised straight-line epilogue — residual fetched by TMA into the output staging slot — whenever the flags are
   * bias[+relu|+gelu] or bias+residual with a plain strided residual; the generic epilogue otherwise),
   * -1 = always the generic epilogue.  Both produce bit-identical results. */
  int32_t epilogue;
  /* Storage types (odb_dtype).  in_dtype: views + weight.  out_dtype: out, out2, residual.
   *   (BF16, BF16)  the wgmma tensor-core path described above;
   *   (BF16, F32)   tensor-core path with an fp32 epilogue: out = residual + (acc + bias), residual and out fp32
   *                 (requires bias and residual, no act / out2 / gn / head): the ViT residual stream;
   *   (F32,  F32)   fp32 correctness mode: the same contraction on the FP32 FMA pipe (weight fp32 [n][taps*C]),
   *                 partial sums combined in fp64; bias / act / residual / out2 as above, no gn_partial / head. */
  int32_t in_dtype;
  int32_t out_dtype;
  /* Activation of the out2 copy: ODB_ACT_NONE / ODB_ACT_RELU = relu (ResidualConvUnit's `relu(out)` operand),
   * ODB_ACT_GELU = exact-erf GELU (train mode: out keeps the pre-activation of mlp.fc1 for the backward, out2 feeds fc2). */
  int32_t out2_act;
} odb_conv_gemm_desc;

int odb_conv_gemm(const odb_conv_gemm_desc* desc, void* stream);
/* The tiling odb_conv_gemm will use for `desc`: out4 = {tiles_x, tiles_y, block_n, flags}, flags bit 0 =
 * CTA pair, bit 1 = halo mode. */
int odb_conv_gemm_plan(const odb_conv_gemm_desc* desc, int32_t* out4);

/* The fp8 inference mode's ViT linear layers (nn.Linear in timm Attention/Mlp, loop M/vit.py:150-151: attn.qkv,
 * attn.proj, mlp.fc1, mlp.fc2) on e4m3 wgmma.  desc as for odb_conv_gemm with in_dtype = ODB_DTYPE_E4M3: views[0] and
 * weight are e4m3 (channels and strides multiples of 16), one view, one tap at offset 0, the input extent equal to
 * the output extent, a bias, no head / halo / CTA pair / gn_partial / out2.  With q_a, q_w the e4m3 operands:
 *   v[r][c] = (sum_k q_a[r][k] * q_w[c][k]) * (row_scale[r] * col_scale[c]) + bias[c]      (fp32, one fma)
 * then the layer's epilogue: bf16 out = act(v) (act NONE or GELU), or fp32 out = residual + v (out_dtype F32,
 * residual fp32).  row_scale fp32 [b][h][w] (one per row of the input), col_scale fp32 [n] (16-byte aligned). */
int odb_conv_gemm_scaled(const odb_conv_gemm_desc* desc, const float* row_scale, const float* col_scale, void* stream);

/* LayerNorm over the last dim (timm Block.norm1/norm2, eps 1e-6): y = (x-mean)/sqrt(var+eps)*g + b.
 * x, y bf16 [rows][cols] (cols multiple of 256, <= 1024); gamma/beta fp32. */
int odb_layernorm(const void* x, const float* gamma, const float* beta, void* y, int64_t rows,
                  int32_t cols, float eps, int32_t x_dtype, int32_t y_dtype, void* stream);
/* odb_layernorm (timm Block.norm1/norm2 in the fp8 inference mode) with an e4m3 output quantised per row from the fp32
 * result z of odb_layernorm's arithmetic: amax = max_k |z[k]|, row_scale = amax / 448, q = cvt.rn.satfinite.e4m3(z *
 * (448 / amax)) (IEEE division); an all-zero row gets row_scale 1 and q 0.  x fp32 or bf16 [rows][cols] (x_dtype),
 * y e4m3 [rows][cols], row_scale fp32 [rows]. */
int odb_layernorm_e4m3(const void* x, const float* gamma, const float* beta, void* y, float* row_scale, int64_t rows,
                       int32_t cols, float eps, int32_t x_dtype, void* stream);
/* The same per-row quantisation of a bf16 tensor: x bf16 [rows][cols] -> y e4m3 [rows][cols], row_scale fp32 [rows];
 * cols in {768, 1024, 3072, 4096}, 16-byte aligned pointers.  Feeds attn.proj from odb_attention's output and mlp.fc2
 * from mlp.fc1's GELU output in the fp8 inference mode (timm Attention.proj / Mlp.fc2 inputs, M/vit.py:150-151). */
int odb_rowquant_e4m3(const void* x, void* y, float* row_scale, int64_t rows, int32_t cols, void* stream);

/* Fused multi-head attention (timm Attention.forward): qkv bf16 [b][tokens][3][heads][64] as written
 * by the qkv linear; out bf16 [b][tokens][heads*64]; softmax(q k^T * scale) v.  wgmma kernel:
 * S and O accumulate in registers, exact two-pass fp32 softmax (global row maximum), P rounded to bf16
 * for the PV product, fp32 row sum of the unrounded P.  tokens <= 4097 (a 64 x 64 patch grid + cls): up to 640
 * tokens K and V of an (image, head) stay resident in shared memory, above that they stream through it per
 * 128-query tile (same arithmetic); more tokens return ODB_ERR_UNSUPPORTED.  lse (optional): fp32
 * [b][heads][tokens] = log2 of the row's sum of exp2(s * scale * log2 e), what odb_attention_bwd re-normalises with
 * (the backward itself takes at most 640 tokens). */
int odb_attention(const void* qkv, void* out, float* lse, int32_t b, int32_t tokens, int32_t heads, float scale,
                  void* stream);
/* fp32 correctness mode of odb_attention: qkv fp32 [b][tokens][3][heads][64], out fp32 [b][tokens][heads*64];
 * dot products and the PV sum in fp64, exp / division exact (no fast-math).  tokens <= 4097. */
int odb_attention_f32(const float* qkv, float* out, int32_t b, int32_t tokens, int32_t heads, float scale,
                      void* stream);

/* fp32 correctness mode of the DPT head tail (M/dpt_depth.py:95-97; the tensor-core path fuses this into
 * odb_conv_gemm's head epilogue): x fp32 [b][h][w][32] = relu(conv3x3 + bias), out[b][k][y][x] = relu?(bias[k] +
 * sum_j w[k][j] x[..j]) fp32 NCHW; `pre` (optional) receives the value before the final ReLU. */
int odb_head_tail_f32(const float* x, const float* w, const float* bias, float* out, float* pre, int32_t b,
                      int32_t h, int32_t wd, int32_t head_c, int32_t relu, void* stream);

/* GroupNorm statistics (timm GroupNormAct, 32 groups), deterministic (no floating-point atomics):
 * stats fp32 [b][groups][2] = (mean, 1/sqrt(var + eps)) over x bf16 [b][hw][c], biased variance,
 * reduced in a fixed order with fp64 combination.  `scratch` is caller-owned device memory of at
 * least odb_groupnorm_scratch_bytes(...) bytes, 256-byte aligned, ZEROED ONCE at allocation (the
 * kernel leaves it zeroed); it may be shared by successive calls on one stream. */
int64_t odb_groupnorm_scratch_bytes(int32_t b, int32_t hw, int32_t c, int32_t groups);
int odb_groupnorm_stats(const void* x, float* stats, void* scratch, int64_t scratch_bytes, int32_t b,
                        int32_t hw, int32_t c, int32_t groups, float eps, int32_t dtype, void* stream);

/* Reduce the partial sums written by odb_conv_gemm (gn_partial) in a fixed order with fp64
 * combination: stats[b][g] = (mean, 1/sqrt(var + eps)); rows_per_image = tiles_x * tiles_y * 4,
 * count = pixels * channels_per_group of one group. */
int odb_groupnorm_finalize(const float* partial, float* stats, int32_t b, int32_t rows_per_image,
                           int32_t groups, double count, float eps, void* stream);

/* GroupNorm apply (+ optional shortcut, + optional ReLU), timm Bottleneck.forward:
 *   y = relu?( gn(x; stats, gamma, beta) + shortcut )
 * shortcut = 0 (res == NULL) | res (res_stats == NULL) | gn(res; res_stats, res_gamma, res_beta). */
int odb_groupnorm_apply(const void* x, const float* stats, const float* gamma, const float* beta,
                        const void* res, const float* res_stats, const float* res_gamma,
                        const float* res_beta, void* y, int32_t b, int32_t hw, int32_t c,
                        int32_t groups, int32_t relu, int32_t dtype, void* stream);

/* Stem tail (timm ResNetV2 stem.norm + stem.pool): GroupNorm+ReLU then MaxPool 3x3 stride 2 with
 * TF-SAME padding (0,1).  x bf16 [b][h][w][c] -> y bf16 [b][h/2][w/2][c]. */
int odb_stem_gn_relu_maxpool(const void* x, const float* stats, const float* gamma,
                             const float* beta, void* y, int32_t b, int32_t h, int32_t w, int32_t c,
                             int32_t groups, int32_t dtype, void* stream);

/* im2col for the 7x7 stride-2 TF-SAME stem conv (timm StdConv2dSame 3->64): x fp32 NCHW
 * [b][3][h][w] -> cols bf16 [b*(h/2)*(w/2)][kpad], column (ky*7+kx)*3+ch, zero padded. */
int odb_stem_im2col(const float* x, void* cols, int32_t b, int32_t h, int32_t w, int32_t kpad,
                    int32_t dtype, void* stream);

/* Bilinear x2 upsampling, align_corners=True (M/blocks.py:335-337, M/dpt_depth.py:93), fused with
 * the skip add of the next fusion block (M/blocks.py:330): out = up2(z) + res; out_relu = relu(out).
 * z bf16 [b][h][w][c]; res/out/out_relu bf16 [b][2h][2w][c]; res and out_relu may be NULL. */
int odb_upsample2x_add(const void* z, const void* res, void* out, void* out_relu, int32_t b,
                       int32_t h, int32_t w, int32_t c, int32_t dtype, void* stream);

/* Patch embedding gather of the plain ViT backbones (DPT-Large `vitl16_384`, `vitb16_384`; timm PatchEmbed =
 * Conv2d(3, D, patch, stride patch), applied at M/vit.py:131): x fp32 NCHW [b][3][h][w] ->
 * cols bf16 [b * (h/patch) * (w/patch)][3 * patch * patch], column (c * patch + py) * patch + px = the row-major
 * flattening of the conv weight, so the embedding is one odb_conv_gemm. */
int odb_patchify(const float* x, void* cols, int32_t b, int32_t h, int32_t w, int32_t patch, int32_t dtype,
                 void* stream);

/* tokens[b][0][:] = cls + pos[0]  (M/vit.py:135-147); tokens bf16 [b][tokens][c]; cls, pos0 fp32 [c]. */
int odb_write_cls_row(void* tokens, const float* cls, const float* pos0, int32_t b, int32_t tokens_n,
                      int32_t c, int32_t dtype, void* stream);

/* ProjectReadout cls term (M/vit.py:43-47): out[b][n] = bias[n] + sum_k w[n][c + k] * tokens[b][0][k]
 * w bf16 [c][2c] (the Linear(2c, c) weight), tokens bf16 [b][tokens][c], out fp32 [b][c]. */
int odb_readout_cls_bias(const void* w, const float* bias, const void* tokens, float* out, int32_t b,
                         int32_t tokens_n, int32_t c, int32_t dtype, void* stream);

/* dst bf16[n] = round(src fp32[n]) (n a multiple of 8): the hooked ViT activations (M/vit.py:158-165 `get_activation`)
 * leave the fp32 residual stream as bf16 operands of the readout GEMM. */
int odb_cast_f32_bf16(const float* src, void* dst, int64_t n, void* stream);

/* =====================================================================================================
 * Backward of the network (train_depth.py:183-190 training_step -> loss.backward(); PL runs autograd over
 * the reference modules).  dgrad of every conv / linear layer is odb_conv_gemm itself with the re-packed
 * (in/out swapped, 180-degree rotated) weight from odb_pack_weight; the entry points below are the rest.
 * `dtype` is the storage type of activations and activation gradients; statistics, affine parameters,
 * parameter gradients and the ViT residual-stream gradient are fp32.  All reductions have a fixed order.
 * ===================================================================================================== */

/* Weight gradient of a convolution / linear layer described like odb_conv_gemm (views + taps):
 *   out[n][t * C + c] (+)= sum_{b,y,x} dy[b,y,x,n] * view[tap_view[t]][b, y + tap_dy[t], x + tap_dx[t], c]
 * i.e. the gradient in the PACKED weight layout of odb_conv_gemm (fp32).  bf16: wgmma kernel with both
 * operands MN-major straight from the channels-last tensors (the 128-byte-swizzled TMA box of 64 pixels x 64
 * channels that feeds the forward as a K-major A tile IS the MN-major operand of the transposed product),
 * split over the pixel range, fp32 partials in `workspace`, ordered reduction.  fp32: FP32-pipe twin. */
typedef struct odb_wgrad_desc {
  int32_t num_views;
  odb_view views[ODB_MAX_VIEWS];
  int32_t num_taps;
  int8_t tap_view[ODB_MAX_TAPS];
  int8_t tap_dx[ODB_MAX_TAPS];
  int8_t tap_dy[ODB_MAX_TAPS];
  odb_view dy;            /* c = n; w, h, b = the layer's output extent */
  int32_t n;
  float* out;             /* fp32 [n][num_taps * C] */
  void* workspace;        /* split partials */
  int64_t workspace_bytes;
  int32_t accumulate;     /* add to `out` instead of overwriting */
  int32_t dtype;          /* odb_dtype of views and dy */
} odb_wgrad_desc;
int64_t odb_conv_wgrad_workspace_bytes(const odb_wgrad_desc* desc);
int odb_conv_wgrad(const odb_wgrad_desc* desc, void* stream);

/* Backward of odb_attention (timm Attention.forward): dqkv [b][tokens][3][heads][64] from qkv, the forward output o
 * [b][tokens][heads*64], its gradient d_o, and (bf16 path) the per-row log2-sum-exp `lse` fp32 [b][heads][tokens]
 * that odb_attention wrote.  bf16: P and dS are re-materialised per (image, head) by wgmma GEMMs with fused
 * softmax / dS epilogues, dQ / dK / dV are three more batched GEMMs; fp32: FP32-pipe twin (lse unused). */
int64_t odb_attention_bwd_workspace_bytes(int32_t b, int32_t tokens, int32_t heads, int32_t dtype);
int odb_attention_bwd(const void* qkv, const void* o, const void* d_o, const float* lse, void* dqkv, void* workspace,
                      int64_t workspace_bytes, int32_t b, int32_t tokens, int32_t heads, float scale, int32_t dtype,
                      void* stream);

/* out = a + b * [mask > 0]   (a, mask optional): ReLU backward and gradient accumulation; n elements (multiple of 8). */
int odb_mask_add(const void* a, const void* b, const void* mask, void* out, int64_t n, int32_t dtype, void* stream);
/* exact-erf GELU (nn.GELU() default) forward on a stored pre-activation, and its backward du = dy * gelu'(u). */
int odb_gelu_fwd(const void* u, void* y, int64_t n, int32_t dtype, void* stream);
int odb_gelu_bwd(const void* dy, const void* u, void* du, int64_t n, int32_t dtype, void* stream);
/* Bias gradients: out[bt][n] (+)= sum over rows of x[bt][row][n] (row / batch strides in elements). */
int64_t odb_colsum_workspace_bytes(int32_t batches, int64_t rows_per_batch, int32_t n);
int odb_colsum(const void* x, float* out, void* workspace, int32_t batches, int64_t rows_per_batch, int32_t n,
               int64_t row_stride, int64_t batch_stride, int32_t accumulate, int32_t dtype, void* stream);
/* out[bt][i] (+)= sum_p partial[bt][p][i] in fp64, in a fixed order (8 interleaved part lanes, then the lanes). */
int odb_reduce_partials(const float* partial, float* out, int32_t batches, int32_t parts, int64_t n, int32_t accumulate,
                        void* stream);
/* LayerNorm backward on the fp32 residual stream: ds_out = ds_in + dLN(dy; x, gamma) (ds_in may be NULL), optional
 * copy of ds_out in `dtype` (the next GEMM operand), dgamma / dbeta (+)=, and optionally (dcolsum != NULL) the column
 * sums of ds_out (+)= : the bias gradient of the linear layer whose output gradient ds_out is (timm Block: attn.proj
 * after norm2's backward, the previous block's mlp.fc2 after norm1's).  dgamma = dbeta = NULL (both or neither): a frozen
 * norm, no affine gradients and no reduction of them — one pass writing ds_out / ds_copy (and dcolsum if given). */
int64_t odb_layernorm_bwd_workspace_bytes(int32_t cols);
int odb_layernorm_bwd(const void* dy, const float* x, const float* gamma, const float* ds_in, float* ds_out, void* ds_copy,
                      float* dgamma, float* dbeta, float* dcolsum, void* workspace, int64_t rows, int32_t cols, float eps,
                      int32_t accumulate, int32_t dtype, void* stream);
/* GroupNorm backward (timm GroupNormAct): g = dy * [mask > 0] (mask NULL: g = dy; the mask is the stored output of the
 * ReLU that follows the norm); dx, dgamma (+)=, dbeta (+)= from x and the forward statistics (mean, rstd).
 * dgamma = dbeta = NULL (both or neither): dx only (the group sums dx needs are still formed). */
int64_t odb_groupnorm_bwd_workspace_bytes(int32_t b, int32_t hw, int32_t c, int32_t groups);
int odb_groupnorm_bwd(const void* dy, const void* mask, const void* x, const float* stats, const float* gamma, void* dx,
                      float* dgamma, float* dbeta, void* workspace, int32_t b, int32_t hw, int32_t c, int32_t groups,
                      int32_t accumulate, int32_t dtype, void* stream);
/* Adjoint of odb_upsample2x_add's bilinear part: dz [b][h][w][c] from dout [b][2h][2w][c]. */
int odb_upsample2x_bwd(const void* dout, void* dz, int32_t b, int32_t h, int32_t w, int32_t c, int32_t dtype, void* stream);
/* Backward of odb_stem_gn_relu_maxpool down to the GroupNorm output: g_s0 [b][h][w][c] = gradient w.r.t. gn(s0), already
 * masked by the ReLU; the pooling gradient goes to the first maximum of each window (torch semantics). */
int odb_stem_pool_bwd(const void* dt, const void* s0, const float* stats, const float* gamma, const float* beta, void* g_s0,
                      int32_t b, int32_t h, int32_t w, int32_t c, int32_t groups, int32_t dtype, void* stream);
/* Gradient w.r.t. the network's input image: replaces autograd's input gradient of the hybrid stem's timm
 * StdConv2dSame(3, 64, 7, stride 2) (TF-SAME padding (2, 3)).  ds0 `dtype` [b][h/2][w/2][64] = gradient w.r.t. the
 * convolution's output, weight `dtype` [64][kpad] = the packed, standardised operand the forward used (column
 * (ky*7+kx)*3+ch, odb_stem_im2col's order) -> dx fp32 NCHW [b][3][h][w], written (not accumulated).  Gather form with a
 * fixed summation order: bit-reproducible and independent of the batch.  h, w even; kpad a multiple of 8 in
 * [152, 1024]; ds0 16-byte and dx 8-byte aligned. */
int odb_stem_input_grad(const void* ds0, const void* weight, float* dx, int32_t b, int32_t h, int32_t w, int32_t kpad,
                        int32_t dtype, void* stream);
/* Gradient w.r.t. the network's input image of the plain-ViT patch embedding: replaces autograd's input gradient of timm
 * PatchEmbed.proj = Conv2d(3, D, patch, stride patch) (modules/midas/vit.py:131); the adjoint of odb_patchify.
 * dcols `dtype` [b * (h/patch) * (w/patch)][3 * patch * patch] (column (c * patch + py) * patch + px) -> dx fp32 NCHW
 * [b][3][h][w], written (not accumulated).  The patches do not overlap: every dx element is one dcols element (a
 * permutation, bit-exact).  patch a multiple of 8 dividing h and w; 16-byte aligned pointers. */
int odb_patch_input_grad(const void* dcols, float* dx, int32_t b, int32_t h, int32_t w, int32_t patch, int32_t dtype,
                         void* stream);
/* Gradient of the 24 x 24 position-embedding grid through its resize to a gh x gw patch grid (modules/midas/vit.py:102-116
 * _resize_pos_embed: F.interpolate(mode="bilinear", align_corners=False), torch's index arithmetic): dpos fp32
 * [24*24][d] = the transpose of that map applied to dgrid fp32 [gh*gw][d], written (not accumulated).  Gather form with a
 * fixed summation order: bit-reproducible.  gh, gw >= 1; d a multiple of 4; 16-byte aligned pointers. */
int odb_pos_embed_resize_bwd(const float* dgrid, float* dpos, int32_t gh, int32_t gw, int32_t d, void* stream);
/* DPT head tail, unfused (training): out[b][k][y][x] = relu?(bias[k] + sum_j w[k][j] a[b][y][x][j]), a has
 * channel_stride channels per pixel of which the first 32 are used; and its backward (da zero in the padding channels;
 * dw = dbias = NULL, both or neither: da only). */
int odb_head_tail_fwd(const void* a, int32_t channel_stride, const float* w, const float* bias, float* out, int32_t b,
                      int32_t h, int32_t wd, int32_t head_c, int32_t relu, int32_t dtype, void* stream);
int64_t odb_head_tail_bwd_workspace_bytes(int32_t head_c);
int odb_head_tail_bwd(const float* dout, const float* out, const void* a, int32_t channel_stride, const float* w, void* da,
                      float* dw, float* dbias, void* workspace, int32_t b, int32_t h, int32_t wd, int32_t head_c,
                      int32_t relu, int32_t accumulate, int32_t dtype, void* stream);
/* ds_out (fp32) = ds_in (fp32, optional) + g (`dtype`); optional copy of ds_out in `dtype`. */
int odb_add_cast(const float* ds_in, const void* g, float* ds_out, void* copy, int64_t n, int32_t dtype, void* stream);
/* train_depth.py:263 `torch.clamp(depth_preds, 0, 1)` and its backward: out = (g1 + g2) * [0 <= p <= 1] (g2 optional). */
int odb_clamp01(const float* p, float* out, int64_t n, void* stream);
int odb_clamp01_bwd(const float* p, const float* g1, const float* g2, float* out, int64_t n, void* stream);
/* Per-step weight packing: w fp32 [n][c][taps] (optionally weight-standardised, timm StdConv2dSame eps) ->
 * fwd `dtype` [n_pad][taps * c_pad] (odb_conv_gemm weight) and bwd `dtype` [c_pad][taps * n_pad] (dgrad weight). */
int odb_pack_weight(const float* w, void* fwd, void* bwd, int32_t n, int32_t c, int32_t taps, int32_t n_pad, int32_t c_pad,
                    int32_t standardize, float eps, int32_t dtype, void* stream);
/* Multi-tensor forms: one launch for a whole table of layers.  `items` is a DEVICE array of n_items records
 *   pack:   { const float* w; void* fwd; void* bwd; int32 n, c, taps, n_pad, c_pad, standardize, first_block, first_tile; }
 *   unpack: { const float* gp; const float* w; float* dw; int32 n, c, taps, c_pad, standardize, first_block, pad, pad; }
 * first_block / first_tile: prefix sums of n_pad (pack rows), ceil(n_pad/32)*ceil(c_pad/32)*taps (transpose tiles), n (unpack
 * rows); total_rows / total_tiles their totals; max_row_floats = max taps * c_pad over the table. */
int odb_pack_weights_multi(const void* items, int32_t n_items, int32_t total_rows, int32_t total_tiles, float eps, int32_t dtype,
                           void* stream);
int odb_unpack_wgrads_multi(const void* items, int32_t n_items, int32_t total_rows, int32_t max_row_floats, float eps,
                            void* stream);
/* Packed-layout weight gradient gp fp32 [n][taps * c_pad] -> parameter layout dw fp32 [n][c][taps], through the weight
 * standardisation when `standardize` (w = the fp32 parameter). */
int odb_unpack_wgrad(const float* gp, const float* w, float* dw, int32_t n, int32_t c, int32_t taps, int32_t c_pad,
                     int32_t standardize, float eps, void* stream);

/* ---- depth-training losses (train_depth.py:261-279), forward and (odb_*_bwd) backward with respect to the
 * prediction; all tensors fp32 [b][h][w] ------- */

/* make_valid_mask (train_depth.py:215-242): valid = nearest_upsample(max_pool2d(1 - mask, pool)) == 0. */
int odb_make_valid_mask(const float* mask_float, uint8_t* mask_valid, int32_t b, int32_t h, int32_t w,
                        int32_t pool, void* stream);

/* MidasLoss(alpha, scales, reduction='image-based').forward (losses/midas_loss.py:137-157):
 * out3 = (total, ssi, reg).  mask: uint8, 1 = valid.  Exact lower nanmedian by radix select,
 * deterministic fp64-combined reductions.  workspace: >= odb_midas_loss_workspace_bytes(b), 256-B aligned. */
int64_t odb_midas_loss_workspace_bytes(int32_t b);
int odb_midas_loss_fwd(const float* prediction, const float* target, const uint8_t* mask, int32_t b,
                       int32_t h, int32_t w, float alpha, int32_t scales, float* out3, void* workspace,
                       int64_t workspace_bytes, void* stream);

/* VNL_Loss.forward(first, second, select) (losses/virtual_normal_loss.py:151-194) for given point
 * triplets p1/p2/p3 (device int32 [n_points], flat index y*w + x — the reference draws them with host
 * NumPy RNG, :52-72).  `first` takes the reference's `gt_depth` slot (train_depth.py:272 passes the
 * PREDICTION there).  group_loss: scratch fp32 [b * n_points]; out1: the scalar loss. */
int odb_vnl_loss_fwd(const float* first, const float* second, const int32_t* p1, const int32_t* p2,
                     const int32_t* p3, int32_t n_points, int32_t b, int32_t h, int32_t w, float fx, float fy,
                     float delta_z, int32_t select, float* out1, float* group_loss, void* stream);

/* Backward of MidasLoss: grad[b][h][w] = d(w_ssi * ssi + w_reg * reg) / d(prediction) exactly as autograd derives it
 * for losses/midas_loss.py:137-157 (ssi through the median element and the deviation; reg through prediction_ssi AND
 * through the least-squares scale / shift).  Call after odb_midas_loss_fwd on the SAME prediction / target / mask with
 * its workspace untouched (fwd_workspace).  For train_depth.py:276 `ssi + 0.1 * reg`: w_ssi = 1, w_reg = 0.1.
 * bwd_workspace: odb_midas_loss_bwd_workspace_bytes(b) bytes; gbuf: scratch fp32 [b][h][w].  Deterministic. */
int64_t odb_midas_loss_bwd_workspace_bytes(int32_t b);
int odb_midas_loss_bwd(const float* prediction, const float* target, const uint8_t* mask, int32_t b, int32_t h,
                       int32_t w, int32_t scales, float w_ssi, float w_reg, const void* fwd_workspace,
                       void* bwd_workspace, float* gbuf, float* grad, void* stream);

/* Backward of VNL_Loss.forward(first, second) with respect to `first` (train_depth.py:272: the prediction):
 * grad fp32 [b][h][w] = upstream * d(loss)/d(first).  Call after odb_vnl_loss_fwd with the same arguments and its
 * group_loss untouched.  acc: scratch, 8 bytes per pixel (64-bit fixed-point accumulators: the scatter over points
 * sampled with replacement is bit-reproducible); sel4: scratch, 4 doubles. */
int odb_vnl_loss_bwd(const float* first, const float* second, const int32_t* p1, const int32_t* p2, const int32_t* p3,
                     int32_t n_points, int32_t b, int32_t h, int32_t w, float fx, float fy, int32_t select,
                     const float* group_loss, float upstream, void* acc, double* sel4, float* grad, void* stream);

/* Normal-training loss pair (SURVEY.md 8(f) rank 2; train_normal.py:247-258): with
 * preds = clamp(prediction, 0, 1) when clamp_prediction != 0,
 *   l1  = masked_l1_loss(preds, target, mask x3)                 (losses/masked_losses.py:4-7)
 *   cos = masked_cosine_angular_loss(preds, target, mask x3)      (losses/masked_losses.py:14-23)
 *   out3 = (cos + 10 * l1, l1, cos).
 * prediction, target fp32 [b][3][h][w]; mask_valid uint8 [b][h][w] (odb_make_valid_mask); workspace: 3 * b doubles.
 * Deterministic (fixed-order fp64 partial sums); backward: odb_normal_loss_bwd. */
int odb_normal_loss_fwd(const float* prediction, const float* target, const uint8_t* mask_valid, int32_t b,
                        int32_t h, int32_t w, int32_t clamp_prediction, float* out3, double* workspace,
                        void* stream);

/* ---- optimizer step of the depth train step (row a21: train_depth.py:381-383 Adam(lr), :425 gradient_clip_val=10)
 * over FLAT fp32 buffers holding all parameters / gradients / moments.
 *
 * odb_clip_grad_norm: torch.nn.utils.clip_grad_norm_(params, max_norm) without the host round trip:
 * out2 = (total L2 norm, clip coefficient min(1, max_norm / (norm + 1e-6))) on the device; the gradients are NOT
 * modified — odb_adam_step applies the coefficient while it reads them.  workspace: odb_grad_norm_workspace_bytes()
 * bytes, 256-byte aligned, zero-filled ONCE by the caller.  Deterministic (fixed-order fp64 partial sums).
 *
 * odb_adam_step: torch.optim.Adam update (betas, eps as given; no weight decay, no amsgrad), step = 1, 2, …;
 * clip2 = the out2 of odb_clip_grad_norm or NULL (no clipping).  step_scalars (device fp32 [2], may be NULL): when given,
 * the two step-dependent scalars (lr / (1 - beta1^step), sqrt(1 - beta2^step)) are read from device memory instead of
 * being computed from `step` — what a CUDA-graph replay of the train step needs; odb_adam_step_scalars (host function,
 * host pointer) computes them exactly as odb_adam_step does.
 *
 * The _segments variants restrict both to the elements of a device table segments int64 [num_segments][2] of [start, end)
 * ranges of the flat buffers (1..1024 disjoint ranges, 16-byte aligned table; every start a multiple of 4, every length but
 * the last a multiple of 4; total = the sum of the lengths): the norm of those gradients only, and no other element of
 * params / exp_avg / exp_avg_sq is read or written.  One launch each, no host synchronisation (CUDA-graph capturable).
 * odb_clip_grad_norm / odb_adam_step are the one-segment case [0, n) of the same kernels. */
int64_t odb_grad_norm_workspace_bytes(void);
int odb_clip_grad_norm(const float* grads, int64_t n, float max_norm, void* workspace, float* out2, void* stream);
int odb_clip_grad_norm_segments(const float* grads, const int64_t* segments, int32_t num_segments, int64_t total,
                                float max_norm, void* workspace, float* out2, void* stream);
int odb_adam_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, int64_t n,
                  const float* clip2, float lr, float beta1, float beta2, float eps, int64_t step,
                  const float* step_scalars, void* stream);
int odb_adam_step_segments(float* params, const float* grads, float* exp_avg, float* exp_avg_sq, const int64_t* segments,
                           int32_t num_segments, int64_t total, const float* clip2, float lr, float beta1, float beta2,
                           float eps, int64_t step, const float* step_scalars, void* stream);
int odb_adam_step_scalars(float lr, float beta1, float beta2, int64_t step, float* out2_host);

/* ---- 3-D refocus augmentation (SURVEY.md 8(f) rank 4; data/refocus_augmentation.py) ------------------------------
 * odb_refocus_quantiles: compute_quantiles (:82-87): quantile_vals fp32 [b][n_quantiles + 1] = torch.quantile(depth[b],
 * i / n_quantiles) (linear interpolation; exact order statistics by radix select), first -= eps, last += eps.
 * odb_refocus_compose: refocus_image (:144-157) after the blur radii are known: the Gaussian blur stack
 * (separable, replicate padding, cutoff int(3 r) made odd, r < 0.1 = copy; radii fp32 [b][levels]) and the per-pixel
 * blend of the two levels bracketing the pixel's depth with weights 1 - dist^2.  rgb fp32 [b][3][h][w], depth fp32
 * [b][h][w], out fp32 [b][3][h][w]; stack_tmp / stack: scratch fp32 [b][levels][3][h][w] each; segments (optional)
 * int32 [b][h][w] = the left quantile index (`return_segments`). */
int odb_refocus_quantiles(const float* depth, int32_t b, int32_t h, int32_t w, int32_t n_quantiles, float eps,
                          float* quantile_vals, void* stream);
int odb_refocus_compose(const float* rgb, const float* depth, const float* quantile_vals, const float* blur_radii,
                        int32_t b, int32_t h, int32_t w, int32_t levels, float* stack_tmp, float* stack, float* out,
                        int32_t* segments, void* stream);

/* Backward of the normal-training loss pair: grad fp32 [b][3][h][w] = d(w_l1 * l1 + w_cos * cos) / d(prediction)
 * (through the clamp when clamp_prediction != 0); for train_normal.py:258 `cos + 10 * l1`: w_l1 = 10, w_cos = 1.
 * fwd_workspace: the workspace odb_normal_loss_fwd filled for the same inputs. */
int odb_normal_loss_bwd(const float* prediction, const float* target, const uint8_t* mask_valid, int32_t b, int32_t h,
                        int32_t w, int32_t clamp_prediction, float w_l1, float w_cos, const double* fwd_workspace,
                        float* grad, void* stream);

int odb_fill_zero(void* ptr, int64_t bytes, void* stream);

/* ---- image pre- / post-processing either side of the forward (SURVEY.md 8(f) rank 1) ------------
 *
 * odb_pil_resize_crop_to_tensor replaces transforms.Resize(384, BILINEAR) + CenterCrop(384) + ToTensor
 * [+ Normalize(0.5, 0.5)] of omnidata_tools/torch/demo.py:74-76,92-95 for an 8-bit image already on the
 * device (src: uint8 [src_h][src_w][channels], channels 1 or 3, row pitch src_pitch bytes).  Pillow's
 * resize is an antialiased two-pass triangle filter in 8-bit fixed point (ImagingResample, 22 fractional
 * bits, 8-bit intermediate); the kernels evaluate exactly that, so `out` is bit-identical to the
 * reference's input tensor.  The host supplies Pillow's coefficient tables restricted to the crop
 * window (omnidata_b200/imageproc.py): bounds_* int32 [n][2] = (first source index, tap count),
 * kk_* int32 [n][ksize_*] fixed-point weights; bounds_h / kk_h for the out_w kept columns, bounds_v / kk_v
 * for the out_h kept rows; the horizontal pass runs over source rows [row0, row0 + nrows) into
 * tmp (uint8 [nrows][out_w][channels]).  out: fp32 [3][out_h][out_w] = (u8 / 255 [- mean) / std]
 * (a single channel is replicated, demo.py:137-138); out_u8 (optional): the cropped 8-bit image. */
int odb_pil_resize_crop_to_tensor(const void* src, int32_t src_h, int32_t src_w, int32_t channels,
                                  int64_t src_pitch, const int32_t* bounds_h, const int32_t* kk_h,
                                  int32_t ksize_h, const int32_t* bounds_v, const int32_t* kk_v, int32_t ksize_v,
                                  int32_t row0, int32_t nrows, int32_t out_h, int32_t out_w, int32_t normalize,
                                  float mean, float stdv, void* tmp, float* out, void* out_u8, void* stream);

/* F.interpolate(x, (out_h, out_w), mode='bicubic') on fp32 planes [planes][in_h][in_w] (align_corners
 * False, A = -0.75) with the clamps of demo.py:140-145 fused: flags bit 0 = clamp the input to [0,1],
 * bit 1 = clamp the result to [0,1], bit 2 = 1 - result. */
int odb_bicubic_resize_f32(const float* in, int32_t planes, int32_t in_h, int32_t in_w, int32_t out_h,
                           int32_t out_w, int32_t flags, float* out, void* stream);

/* F.interpolate(x, (out_h, out_w), mode='bilinear', align_corners=False, antialias=True) on fp32 planes
 * [planes][in_h][in_w] -> out [planes][out_h][out_w]: a separable triangle filter whose support scales with the
 * downsampling factor (plain bilinear when upsampling), horizontal pass into tmp fp32 [planes][in_h][out_w], then
 * vertical.  Per axis the host passes bounds int32 [out][2] = (first input index, tap count) and weights fp32
 * [out][ksize] normalised to sum 1 (omnidata_b200/imageproc.py bilinear_aa_weights: Pillow's coefficients before the
 * 8-bit step).  fp32 fused multiply-adds in tap order; deterministic.  planes, in_h, out_h <= 65535. */
int odb_resize_bilinear_f32(const float* in, int32_t planes, int32_t in_h, int32_t in_w, int32_t out_h, int32_t out_w,
                            const int32_t* bounds_h, const float* weights_h, int32_t ksize_h, const int32_t* bounds_v,
                            const float* weights_v, int32_t ksize_v, float* tmp, float* out, void* stream);

/* transforms.ToPILImage() on a float CHW tensor (demo.py:150): out uint8 [h][w][c] = trunc(x * 255);
 * clamp01 != 0 applies the reference's .clamp(0, 1) first (demo.py:140). */
int odb_f32_chw_to_u8_hwc(const float* in, int32_t c, int32_t h, int32_t w, int32_t clamp01, void* out,
                          void* stream);

/* ---- tiled inference: merging overlapping tile predictions (omnidata_b200/tiled.py TiledPredictor) ------------
 *
 * The reference predicts one 384 x 384 crop per image (demo.py:74-76 Resize + CenterCrop, then DPT.forward,
 * M/dpt_depth.py:67-85,107).  These entry points cut an image of any size into tiles the forward accepts and merge the
 * tiles' predictions back at the image's own size.  Tile grid per axis (length L, tile t, overlap v, 0 <= 2 v < t):
 * L <= t: one tile at 0; else n = ceil((L - v) / (t - v)) tiles at o_k = round(k (L - t) / (n - 1)), halves rounded up.
 * Tiles are numbered row-major (i = ty * nx + tx, T = ny * nx <= ODB_TILE_MAX_TILES per image).  Pairs: the ny (nx - 1)
 * horizontal neighbour pairs row-major, then the (ny - 1) nx vertical ones; "a" is the left / upper tile's prediction,
 * "b" the other's.  tile_h, tile_w: multiples of 32; b, h, w <= 65535.
 *
 * odb_tile_gather: tiles fp32 [b * T][3][tile_h][tile_w] (16-byte aligned) from image fp32 [b][3][h][w], replicating
 * the last row / column where the image is smaller than a tile.
 * odb_tile_overlap_moments (depth): moments fp64 [b][pairs][6] = (n, Sa, Sb, Saa, Sbb, Sab) over each pair's overlap
 * inside the image, from pred fp32 [b * T][tile_h][tile_w]; no launch for a single tile.
 * odb_tile_align_solve (depth): scale_shift fp64 [b][T][2] = (s_i, t_i) minimising
 *   sum_pairs sum_overlap (s_i a + t_i - s_j b - t_j)^2 + 1e-3 Nbar sum_i ((s_i - 1)^2 + t_i^2)
 * (Nbar = the mean overlap pixel count, at least 1) — the per-image scale-and-shift least squares of
 * L/midas_loss.py:10-30 (compute_scale_and_shift) solved for all tiles of an image jointly.  Banded fp64 Cholesky, one
 * CTA per image; workspace: odb_tile_align_workspace_bytes(b, tiles_y, tiles_x) bytes (0: none needed; negative:
 * refused).  moments may be NULL for a single tile.
 * odb_tile_blend: out fp32 [b][c][h][w] (the forward's output layout) = sum_i w_i (s_i d_i + t_i) / sum_i w_i over the
 * tiles covering each pixel, row-major, fp32; pred fp32 [b * T][c][tile_h][tile_w]; scale_shift NULL: s = 1, t = 0.
 * w_i = rho(dy) rho(dx), rho(d) = min(1, (d + 1) / (overlap + 1)), d = the distance to the tile's nearest edge that is
 * not on the image border.
 * odb_tile_anchor_moments (depth, anchored): moments fp64 [b][T][5] = (n, Sa, Saa, Sg, Sag) over each tile's pixels
 * inside the image (n = min(tile_h, h) min(tile_w, w)), a from pred fp32 [b * T][tile_h][tile_w], g from anchor fp32
 * [b][h][w] (a whole-image prediction resampled to h x w).
 * odb_tile_align_solve_anchored (depth): scale_shift as odb_tile_align_solve, minimising
 *   sum_pairs sum_overlap (s_i a + t_i - s_j b - t_j)^2 + 1e-3 Nbar sum_i (1 / n_i) sum_tile (s_i a + t_i - g)^2
 *   + 1e-6 1e-3 Nbar sum_i ((s_i - 1)^2 + t_i^2)
 * — each tile anchored to g with the weight the ridge carries in odb_tile_align_solve, the ridge kept at 1e-6 of it so
 * that a flat tile stays well-posed.  Same band, workspace and tile cap; anchor_moments (from odb_tile_anchor_moments)
 * is required, moments may be NULL for a single tile, which then gets compute_scale_and_shift of the tile against g.
 * All are deterministic and batch-independent. */
#define ODB_TILE_MAX_TILES 1024
int odb_tile_gather(const float* image, int32_t b, int32_t h, int32_t w, int32_t tile_h, int32_t tile_w,
                    int32_t overlap, float* tiles, void* stream);
int odb_tile_overlap_moments(const float* pred, int32_t b, int32_t h, int32_t w, int32_t tile_h, int32_t tile_w,
                             int32_t overlap, double* moments, void* stream);
int64_t odb_tile_align_workspace_bytes(int32_t b, int32_t tiles_y, int32_t tiles_x);
int odb_tile_align_solve(const double* moments, int32_t b, int32_t tiles_y, int32_t tiles_x, void* workspace,
                         double* scale_shift, void* stream);
int odb_tile_blend(const float* pred, const double* scale_shift, int32_t b, int32_t c, int32_t h, int32_t w,
                   int32_t tile_h, int32_t tile_w, int32_t overlap, float* out, void* stream);
int odb_tile_anchor_moments(const float* pred, const float* anchor, int32_t b, int32_t h, int32_t w, int32_t tile_h,
                            int32_t tile_w, int32_t overlap, double* moments, void* stream);
int odb_tile_align_solve_anchored(const double* moments, const double* anchor_moments, int32_t b, int32_t tiles_y,
                                  int32_t tiles_x, void* workspace, double* scale_shift, void* stream);

/* ---- evaluation metrics against ground truth (omnidata_b200/metrics.py DepthMetrics / NormalMetrics) ------------
 *
 * No reference counterpart: the reference monitors its training losses only.  Definitions in DESIGN.md §3
 * "Evaluation metrics"; oracle/metrics_oracle.py restates them in float64.  Inputs are fp32, [b][h][w] per plane;
 * mask: NULL with ODB_MASK_NONE, or uint8 / fp32 [b][h][w] (nonzero = valid) with ODB_MASK_U8 / ODB_MASK_F32.
 * b <= 65535, h, w <= 65535.  Per-pixel arithmetic is fp64.  Every image is cut into fixed pixel slabs, combined in a
 * fixed order and folded into the running state image after image, in image order: the state after a dataset does not
 * depend on how it was split into batches, and repeat runs give the same bits (no floating-point atomics).  The state
 * buffers are the caller's, zeroed to start.  workspace: odb_metrics_workspace_bytes(b, h, w) bytes, 8-byte aligned
 * (negative: refused).  Arguments are checked before any launch.
 *
 * odb_depth_metrics_update: pred, gt (depth) fp32 [b][h][w].  Valid set of an image V = {mask != 0, gt finite,
 * gt > min_depth, gt <= max_depth}; max_depth = +inf means none (required finite in disparity space), 0 <= min_depth <
 * max_depth.  Per image, (s, t) is the least-squares fit over V of s p + t to y, with the five fp64 moments and the
 * convention of L/midas_loss.py:10-30 compute_scale_and_shift (s = t = 0 where det <= 0):
 *   ODB_SPACE_DEPTH:     y = gt,     dh = clamp(s p + t, min_depth, max_depth)
 *   ODB_SPACE_DISPARITY: y = 1 / gt, dh = clamp(1 / max(s p + t, 1 / max_depth), min_depth, max_depth)
 * and over V, with e = dh - gt, r = max(dh / gt, gt / dh):  AbsRel = mean |e| / gt, SqRel = mean e^2 / gt,
 * RMSE = sqrt(mean e^2), RMSE_log = sqrt(mean (ln dh - ln gt)^2), delta_k = #(r < 1.25^k) / |V|.
 * records fp64 [b][ODB_DEPTH_RECORD] = (|V|, AbsRel, SqRel, RMSE, RMSE_log, #delta1, #delta2, #delta3, s, t, det <= 0,
 * non-finite predictions on V); a non-finite prediction on V makes the image's metrics NaN.  Images with |V| > 0 add
 * state_sums fp64 [7] += (AbsRel, SqRel, RMSE, RMSE_log, delta1, delta2, delta3) and state_counts int64 [4] +=
 * (1, 0, det <= 0, |V|); images with |V| = 0 add (0, 1, 0, 0).  Five launches.
 *
 * odb_normal_metrics_update: pred, gt fp32 [b][3][h][w] in the model's output encoding [0, 1].  Per pixel, a = 2 pred - 1,
 * g = 2 gt - 1, theta = atan2(|a x g|, a . g) in degrees; the pixel takes part where the mask is nonzero and |a|, |g| >
 * 1e-6.  state_sums fp64 [2] += (S theta, S theta^2), state_counts int64 [5] += (#finite theta, #non-finite theta,
 * #(theta < 11.25), #(theta < 22.5), #(theta < 30)) over the finite ones, and hist int64 [ODB_NORMAL_HIST_BINS] (bins of
 * 1 / ODB_NORMAL_HIST_PER_DEGREE degree) += 1 at floor(4096 theta) (integer atomics).  Three launches.
 * odb_normal_metrics_median: out fp64 [2] = (k, (k + 0.5) / 4096) for the bin k holding the 0-based rank
 * floor((N - 1) / 2) of the N angles counted in hist (the lower median to 2^-13 degree); (-1, NaN) for N = 0. */
#define ODB_MASK_NONE 0
#define ODB_MASK_U8 1
#define ODB_MASK_F32 2
#define ODB_SPACE_DEPTH 0
#define ODB_SPACE_DISPARITY 1
#define ODB_DEPTH_RECORD 12
#define ODB_NORMAL_HIST_PER_DEGREE 4096
#define ODB_NORMAL_HIST_BINS (180 * ODB_NORMAL_HIST_PER_DEGREE + 1)
int64_t odb_metrics_workspace_bytes(int32_t b, int32_t h, int32_t w);
int odb_depth_metrics_update(const float* pred, const float* gt, const void* mask, int32_t mask_dtype, int32_t b,
                             int32_t h, int32_t w, int32_t space, double min_depth, double max_depth, void* workspace,
                             double* records, double* state_sums, int64_t* state_counts, void* stream);
int odb_normal_metrics_update(const float* pred, const float* gt, const void* mask, int32_t mask_dtype, int32_t b,
                              int32_t h, int32_t w, void* workspace, double* state_sums, int64_t* state_counts,
                              int64_t* hist, void* stream);
int odb_normal_metrics_median(const int64_t* hist, double* out, void* stream);
/* odb_depth_metrics_update_metric: odb_depth_metrics_update in depth space without the fit, for predictions that are
 * already metric (a sparse alignment's output): dh = clamp(pred, min_depth, max_depth), and the records hold s = 1,
 * t = 0, det <= 0 never.  Five launches. */
int odb_depth_metrics_update_metric(const float* pred, const float* gt, const void* mask, int32_t mask_dtype,
                                    int32_t b, int32_t h, int32_t w, double min_depth, double max_depth,
                                    void* workspace, double* records, double* state_sums, int64_t* state_counts,
                                    void* stream);

/* ---- sparse metric alignment (omnidata_b200/sparse.py SparseDepthAligner) -----------------------------------------
 *
 * No reference counterpart.  Maps an affine-invariant depth prediction to metres with scale and shift fields fitted to
 * sparse measured depths (LiDAR returns, SfM points).  Definitions in DESIGN.md §3 "Sparse metric alignment";
 * oracle/sparse_oracle.py restates them in float64.  pred, sparse fp32 [b][h][w] (sparse in metres, 0 / NaN = none);
 * mask as for the metrics above; b, h, w <= 65535.  Points V = {mask != 0, sparse finite, min_depth < sparse <=
 * max_depth}, y = sparse (ODB_SPACE_DEPTH) or 1 / sparse (ODB_SPACE_DISPARITY, max_depth finite); max_depth = +inf:
 * none, 0 <= min_depth < max_depth.
 *
 * Fields: nodes fp64 [b][grid_y][grid_x][2] = (s_i, t_i), 1 <= grid_y <= h, 1 <= grid_x <= w, grid_y grid_x <=
 * ODB_SPARSE_MAX_NODES.  S(p), T(p) = the bilinear resize of the node maps to h x w (align_corners=False, no
 * antialiasing): u = ((x + 0.5) grid_x) / w - 0.5 clamped to [0, grid_x - 1], likewise along y, in fp64 round-to-nearest
 * operations.  z_p = S(p) a_p + T(p).  The fit minimises
 *   E = S_V w_p (z_p - y_p)^2 + smooth (n / n_e) S_{i~j} mean_V((s_i - s_j) a_p + (t_i - t_j))^2
 * over the n_e 4-neighbour node edges (n = |V|; smooth finite >= 0, > 0 when there is more than one node).
 * robust = 0: one solve with w = 1 (iterations = 1).  robust = delta > 0: `iterations` in [2, 32] solves, the first with
 * w = 1, each later one with w_p = min(1, delta / |r_p|), r_p = (z_p - y_p) / y_p of the previous solve (Huber IRLS).
 * The normal equations (half-bandwidth 2 grid_x + 3) are solved in fp64 by a banded Cholesky factorisation.
 * records fp64 [b][ODB_SPARSE_RECORD] = (n, status, RMS of r over V for the final nodes, fraction of V with w < 1 in
 * the last solve, 0, 0, 0, 0); status 0 ok, 1 n < 2, 2 degenerate (S w a^2 S w - (S w a)^2 <= 0: all a equal on V),
 * 3 a non-finite prediction on V; for status != 0 the nodes and the residual are NaN.
 *
 * odb_sparse_align_fit: workspace odb_sparse_align_workspace_bytes(b, h, w, grid_y, grid_x) bytes, 8-byte aligned
 * (negative: refused).  3 (iterations + 1) launches.
 * odb_sparse_align_apply: out fp32 [b][h][w] = clamp(z, min_depth, max_depth) (depth space) or clamp(1 / max(z,
 * 1 / max_depth), min_depth, max_depth) (disparity space), computed in fp64 (odb_depth_metrics_update's dh with s = S(p),
 * t = T(p)) and rounded to fp32 once; NaN where a_p is not finite or the nodes are NaN.  S and T are not written to
 * memory.  16-byte accesses where w % 4 == 0 and pred, out are 16-byte aligned.  One launch.
 *
 * No floating-point atomics and fixed partitions: results are bit-reproducible and independent of the batch.  Arguments
 * are checked before any launch. */
#define ODB_SPARSE_MAX_NODES 1024
#define ODB_SPARSE_RECORD 8
int64_t odb_sparse_align_workspace_bytes(int32_t b, int32_t h, int32_t w, int32_t grid_y, int32_t grid_x);
int odb_sparse_align_fit(const float* pred, const float* sparse, const void* mask, int32_t mask_dtype, int32_t b,
                         int32_t h, int32_t w, int32_t grid_y, int32_t grid_x, int32_t space, double min_depth,
                         double max_depth, double smooth, double robust, int32_t iterations, void* workspace,
                         double* nodes, double* records, void* stream);
int odb_sparse_align_apply(const float* pred, const double* nodes, int32_t b, int32_t h, int32_t w, int32_t grid_y,
                           int32_t grid_x, int32_t space, double min_depth, double max_depth, float* out,
                           void* stream);

/* ---- depth-normal fusion (omnidata_b200/fusion.py DepthNormalFusion, depth_normals) ----------------------------
 *
 * No reference counterpart.  Combines a depth prediction with the surface-normal prediction of the same frame.
 * Definitions in DESIGN.md §3 "Depth-normal fusion"; oracle/fusion_oracle.py restates them in float64.
 * depth a fp32 [b][h][w] (z-depth: the clamped relative prediction or metres); normals c fp32 [b][3][h][w] in the
 * normal model's output encoding [0, 1]; mask as for the metrics above; b, h, w <= 65535.  Intrinsics fx, fy > 0, cx,
 * cy finite, in pixels of this resolution, one set for the call.  Pixel (x, y) has the ray r = ((x - cx) / fx,
 * (y - cy) / fy, 1) (OpenCV frame, integer pixel centres).  axis_x, axis_y, axis_z = +-1 map the model's encoding to
 * that frame: n = axes (2 clamp(c, 0, 1) - 1); (1, -1, -1) reads it as x right, y up, z towards the camera.
 * V = {mask != 0, a finite}.  A normal is usable when its three channels are finite and |n| >= 0.5; it is then
 * normalised.  A 4-neighbour edge (p, q) is kept when both ends are in V with usable normals, n_p . n_q > 0 and
 * |a_q - a_p| <= jump (max_V a - min_V a) (jump finite > 0).  Every operation of the coefficients is an fp64
 * round-to-nearest operation.
 *
 * odb_depth_normal_fusion: with m = normalise(n_p + n_q), alpha = m . r_p, beta = m . r_q, e_pq = beta z_q - alpha z_p,
 *   E(z, t) = weight S_V (z - a - t)^2 + weight kappa |V| t^2 + S_kept e_pq^2,   kappa = 1e-6,
 * t = 0 when shift = 0.  Eliminating t leaves M z = weight (z - s(z)) + N z = weight (a - s(a)), s(v) = S_V v /
 * (|V| (1 + kappa)) (s = 0 without shift), solved by Jacobi-preconditioned conjugate gradients in fp64 from z = a.
 * An image stops when |r| <= tol |b| (tol finite > 0) or after `iterations` in [1, 10000]; a stopped image's state is
 * not written again, so the result does not depend on the batch.  weight finite > 0, shift 0 or 1.
 * out fp32 [b][h][w] = z rounded once, NaN off V.  records fp64 [b][ODB_FUSION_RECORD] = (|V|, status, kept edges,
 * iterations run, final |r| / |b|, t, RMS over V of z - a - t, 0); status 0 converged, 1 V empty, 2 a constant on V
 * (1 and 2: output, |r| / |b|, t and RMS NaN), 3 not converged (the output is the last iterate).
 * workspace: odb_fusion_workspace_bytes(b, h, w) bytes (88 per pixel and a small per-image head), 16-byte aligned
 * (negative: refused).  A memset, then 2 iterations + 6 launches, and no host synchronisation; once every image has
 * stopped the remaining launches return after reading one flag.  An edge whose two coefficients are both 0 adds nothing
 * to E and is not counted.
 *
 * odb_depth_normals: out fp32 [b][3][h][w] = the normals of the depth map in the model's encoding.  X = a r on V; an
 * edge is kept when both ends are in V and |a_q - a_p| <= jump (max_V a - min_V a).  t_x = X(x+1) - X(x-1) with both
 * horizontal edges kept, else the one-sided difference over the kept one; t_y likewise.  n = normalise(t_y x t_x),
 * negated when n . X > 0 (facing the camera), out = (axes n + 1) / 2; NaN in all three channels off V or where a tangent
 * is missing.  fp64 round-to-nearest operations, rounded to fp32 once; 16-byte stores where w % 4 == 0 and out is
 * 16-byte aligned.  workspace: odb_depth_normals_workspace_bytes(b, h, w) bytes, 8-byte aligned.  Three launches.
 *
 * No floating-point atomics and fixed partitions: results are bit-reproducible and independent of the batch.  Arguments
 * are checked before any launch. */
#define ODB_FUSION_RECORD 8
int64_t odb_fusion_workspace_bytes(int32_t b, int32_t h, int32_t w);
int64_t odb_depth_normals_workspace_bytes(int32_t b, int32_t h, int32_t w);
int odb_depth_normal_fusion(const float* depth, const float* normals, const void* mask, int32_t mask_dtype, int32_t b,
                            int32_t h, int32_t w, double fx, double fy, double cx, double cy, int32_t axis_x,
                            int32_t axis_y, int32_t axis_z, double jump, double weight, int32_t shift,
                            int32_t iterations, double tol, void* workspace, float* out, double* records,
                            void* stream);
int odb_depth_normals(const float* depth, const void* mask, int32_t mask_dtype, int32_t b, int32_t h, int32_t w,
                      double fx, double fy, double cx, double cy, int32_t axis_x, int32_t axis_y, int32_t axis_z,
                      double jump, void* workspace, float* out, void* stream);

/* ---- TSDF volumes (omnidata_b200/volume.py TSDFVolume) ------------------------------------------------------------
 *
 * No reference counterpart.  Fuses posed depth frames into one dense truncated signed-distance grid, renders depth
 * back from it and extracts a triangle mesh.  Definitions in DESIGN.md §3 "TSDF volumes"; oracle/volume_oracle.py
 * restates them in float64.  Camera frame: OpenCV (x right, y down, z forward, integer pixel centres); intrinsics fx,
 * fy > 0, cx, cy finite, in pixels of the depth map.  A pose cam_to_world is a HOST array of 16 doubles, the row-major
 * 4 x 4 camera-to-world matrix [R t; 0 0 0 1] (finite, last row exactly 0 0 0 1, |R^T R - I| <= 1e-6 entrywise); the
 * entry points read it during the call and pass it to the kernels by value, so the caller copies nothing to the device.
 * Grid: nx, ny, nz in [2, ODB_TSDF_MAX_DIM], nx ny nz <= ODB_TSDF_MAX_POINTS, points X(i, j, k) = origin + voxel (i, j,
 * k) (origin finite, voxel finite > 0).  tsdf, weight fp32 [nz][ny][nx] (i fastest); color NULL or fp32 [3][nz][ny][nx].
 *
 * odb_tsdf_integrate: depth fp32 [b][h][w] in metres with b poses (cam_to_world [b][16]); rgb fp32 [b][3][h][w] exactly
 * when color is given.  Each grid point loops over the b frames in order, in fp64 round-to-nearest operations: Xc =
 * R^T (X - t); no observation when z <= 0; u = fx x / z + cx, v = fy y / z + cy; the pixel (floor(u + 0.5),
 * floor(v + 0.5)) must lie in the image; its depth d must be finite and > 0; eta = d - z, no observation when
 * eta < -trunc (trunc finite > 0); f = min(1, eta / trunc) rounded to fp32.  An observation updates, in fp32 operations,
 * F = (F W + f) / (W + 1), the colour means likewise, then W = W + 1.  One launch per 16 frames; no workspace.
 *
 * odb_tsdf_raycast: out fp32 [h][w] = the z-depth of the first surface along each pixel's ray, 0 where none is hit.  The
 * unit ray R r / |r|, r = ((x - cx) / fx, (y - cy) / fy, 1), from t is clipped to the grid's box [origin, origin + voxel
 * (n - 1)]; samples at t_k = t_enter + k step (step finite in [voxel / 64, voxel]) while t_k <= t_exit are trilinear
 * interpolations of F, valid when all 8 corners have W > 0.  The hit is the first pair of valid samples k, k + 1 with
 * F_k > 0 >= F_k+1 at t_k + step F_k / (F_k - F_k+1); out = that t / |r|.  fp64 round-to-nearest over the fp32 loads.
 * odb_tsdf_raycast_color: the same out, bit for bit, and rgb fp32 [3][h][w] = the colour at the hit, NaN where out = 0:
 * the colour trilinearly interpolated (the same corners and x, y, z order as F) at t_k and at t_k+1, blended as
 * c_k + f (c_k+1 - c_k) with f = F_k / (F_k - F_k+1).  The colour is read only at the hit.
 *
 * odb_tsdf_mesh_count + odb_tsdf_mesh_emit: marching tetrahedra on the Kuhn split of each cell into 6 tetrahedra (one
 * per permutation of the axes).  Each point p owns the 7 lattice edges (p, p + d), d in {0,1}^3 \ {0}, direction index
 * dx + 2 dy + 4 dz - 1; an edge carries a vertex when both ends have W > 0 and exactly one has F < 0, at world position
 * origin + voxel (p + d F_p / (F_p - F_q)) (fp64, stored fp32; colour interpolated likewise).  Vertex ids follow
 * (k, j, i, direction).  A tetrahedron whose 4 corners have W > 0 and 1-3 corners with F < 0 emits 1 or 2 triangles,
 * ordered by (cell, tetrahedron, triangle) and wound by a fixed table so that normals point from F < 0 to F > 0.
 * count: writes counts int64 [2] = (vertices, faces) on the device and the per-point tables to workspace
 * (odb_tsdf_mesh_workspace_bytes(nx, ny, nz) bytes, 8-byte aligned, negative: refused); three launches.  emit: after
 * count on the same workspace, writes vertices fp32 [V][3], faces int32 [F][3] and colors fp32 [V][3] (exactly when
 * color is given); the caller reads the counts and sizes the outputs.  One launch.
 *
 * Integer scans and no atomics: every output is bit-reproducible, and integrating frames in one call or several gives
 * the same bits.  Arguments are checked before any launch. */
#define ODB_TSDF_MAX_DIM 2048
#define ODB_TSDF_MAX_POINTS 268435456
int64_t odb_tsdf_mesh_workspace_bytes(int32_t nx, int32_t ny, int32_t nz);
int odb_tsdf_integrate(float* tsdf, float* weight, float* color, int32_t nx, int32_t ny, int32_t nz, double ox,
                       double oy, double oz, double voxel, double trunc, const float* depth, const float* rgb, int32_t b,
                       int32_t h, int32_t w, double fx, double fy, double cx, double cy, const double* cam_to_world,
                       void* stream);
int odb_tsdf_raycast(const float* tsdf, const float* weight, int32_t nx, int32_t ny, int32_t nz, double ox, double oy,
                     double oz, double voxel, const double* cam_to_world, int32_t h, int32_t w, double fx, double fy,
                     double cx, double cy, double step, float* out, void* stream);
int odb_tsdf_raycast_color(const float* tsdf, const float* weight, const float* color, int32_t nx, int32_t ny,
                           int32_t nz, double ox, double oy, double oz, double voxel, const double* cam_to_world,
                           int32_t h, int32_t w, double fx, double fy, double cx, double cy, double step, float* out,
                           float* rgb, void* stream);
int odb_tsdf_mesh_count(const float* tsdf, const float* weight, int32_t nx, int32_t ny, int32_t nz, void* workspace,
                        int64_t* counts, void* stream);
int odb_tsdf_mesh_emit(const float* tsdf, const float* weight, const float* color, int32_t nx, int32_t ny, int32_t nz,
                       double ox, double oy, double oz, double voxel, const void* workspace, float* vertices,
                       int32_t* faces, float* colors, void* stream);

/* ---- Sparse TSDF volumes (omnidata_b200/volume.py SparseTSDFVolume) ----------------------------------------------
 *
 * No reference counterpart.  The TSDF volume above without a box: definitions in DESIGN.md §3 "Sparse TSDF volumes";
 * oracle/sparse_volume_oracle.py restates them in float64.  Frames, intrinsics and poses as for the TSDF volumes.
 *
 * Lattice: points X(p) = origin + voxel p, p in Z^3, stored in blocks of 8^3: block b holds p = 8 b + (0..7)^3, laid
 * out [k][j][i], with |b| < ODB_SPARSE_TSDF_BLOCK_RANGE per axis.  A block's key packs (bz, by, bx) + RANGE into 21
 * bits each, bz highest, so keys order blocks by (bz, by, bx).  odb_sparse_tsdf describes one volume, all device
 * arrays: data fp32 [capacity][channels][512] (channel 0 F, 1 W, 2-4 the colour means when channels = 5); keys int64
 * [capacity] and birth int32 [capacity] of blocks 0..blocks-1 in id order; nbr int32 [capacity][8], entry c the id of
 * block b + (c & 1, c >> 1 & 1, c >> 2) (-1: unallocated); the hash table table_keys int64 / table_ids int32 /
 * table_birth int32 [table_size] (a power of two >= 1024, -1 / -1 / INT_MAX empty, at most half full between calls);
 * bbox int32 [6] = the allocated blocks' min (x, y, z) and max (x, y, z), (INT_MAX x 3, INT_MIN x 3) when empty;
 * scratch int32 [2 + table_size].
 *
 * Allocation of a call of b frames numbered frame0.. (frames count from the volume's construction or reset):
 * odb_sparse_tsdf_mark: a pixel with finite depth d, 0 < d <= max_depth, covers its ray from z = d - trunc to
 * z = d + trunc; in fp64 round-to-nearest, r = ((x - cx) / fx, (y - cy) / fy), the endpoint at z is X = R (z r_x,
 * z r_y, z) + t, summed in the order x, y, z, then t; its block is floor(((X - origin) / voxel) * 0.125) per axis.  Every
 * block of the box of the two endpoints' blocks is inserted into the table (integer CAS) with the earliest frame that
 * covers it (integer atomicMin); blocks outside the range are not.  scratch[0] = the number of new blocks; scratch[1]
 * = 1 when the table passed half full (the caller doubles the table, rebuilds it and marks again).
 * odb_sparse_tsdf_rebuild: clears the table and inserts blocks 0..blocks-1 with their ids (after growing the table,
 * and to forget a mark that is not committed).
 * odb_sparse_tsdf_commit: gives the n_new marked blocks the ids blocks.. blocks+n_new-1 in the order (birth frame,
 * key), zeroes their data, widens bbox and refreshes nbr; workspace: odb_sparse_tsdf_commit_workspace_bytes(n_new),
 * 16-byte aligned.  capacity >= blocks + n_new.
 * odb_sparse_tsdf_integrate: odb_tsdf_integrate's per-point arithmetic at every point of blocks 0..blocks-1, where a
 * point updates from frame g only when g >= its block's birth frame.
 * odb_sparse_tsdf_raycast: odb_tsdf_raycast (and, with rgb, odb_tsdf_raycast_color) over the grid of bbox: origin
 * lo = origin + voxel 8 bmin, n = 8 (bmax - bmin + 1) points per axis, with unallocated points W = 0.  Samples of
 * unallocated blocks are skipped without changing a bit.  Reads bbox on the device: no synchronisation.
 * odb_sparse_tsdf_mesh_count + _emit: odb_tsdf_mesh_count / _emit over the allocated points (unallocated: W = 0), with
 * vertices at origin + voxel (p + d s), vertex ids in (block id, point, direction) order and faces in (block id, cell,
 * tetrahedron, triangle) order; workspace odb_sparse_tsdf_mesh_workspace_bytes(blocks), 8-byte aligned.
 *
 * Integer atomics only in the table, its birth stamps and the bounding box; every output is bit-reproducible and does
 * not depend on how frames are split into calls. */
#define ODB_SPARSE_TSDF_BLOCK_RANGE 1048576
#define ODB_SPARSE_TSDF_MAX_BLOCKS 2097152
typedef struct {
  float* data;
  int64_t* keys;
  int32_t* birth;
  int32_t* nbr;
  int64_t* table_keys;
  int32_t* table_ids;
  int32_t* table_birth;
  int32_t* bbox;
  int32_t* scratch;
  int32_t blocks, capacity, table_size, channels;
  double ox, oy, oz, voxel;
} odb_sparse_tsdf;
int odb_sparse_tsdf_rebuild(const odb_sparse_tsdf* vol, void* stream);
int odb_sparse_tsdf_mark(const odb_sparse_tsdf* vol, double trunc, double max_depth, const float* depth, int32_t b,
                         int32_t h, int32_t w, double fx, double fy, double cx, double cy, const double* cam_to_world,
                         int32_t frame0, void* stream);
int64_t odb_sparse_tsdf_commit_workspace_bytes(int32_t n_new);
int odb_sparse_tsdf_commit(const odb_sparse_tsdf* vol, int32_t n_new, void* workspace, void* stream);
int odb_sparse_tsdf_integrate(const odb_sparse_tsdf* vol, double trunc, const float* depth, const float* rgb,
                              int32_t b, int32_t h, int32_t w, double fx, double fy, double cx, double cy,
                              const double* cam_to_world, int32_t frame0, void* stream);
int odb_sparse_tsdf_raycast(const odb_sparse_tsdf* vol, const double* cam_to_world, int32_t h, int32_t w, double fx,
                            double fy, double cx, double cy, double step, float* out, float* rgb, void* stream);
int64_t odb_sparse_tsdf_mesh_workspace_bytes(int32_t blocks);
int odb_sparse_tsdf_mesh_count(const odb_sparse_tsdf* vol, void* workspace, int64_t* counts, void* stream);
int odb_sparse_tsdf_mesh_emit(const odb_sparse_tsdf* vol, const void* workspace, float* vertices, int32_t* faces,
                              float* colors, void* stream);

/* ---- camera tracking (omnidata_b200/track.py FrameTracker) ---------------------------------------------------------
 *
 * No reference counterpart.  Solves one frame's camera pose (and, with affine, the scale and shift of its depth) against
 * a model depth map rendered at a reference pose: point-to-plane ICP with projective association (KinectFusion), one
 * Gauss-Newton step per launch.  Definition in DESIGN.md §3 "Camera tracking"; oracle/track_oracle.py restates it in
 * float64.  Frames, intrinsics and poses as for the TSDF volumes above; ref_pose and init_pose are HOST arrays of 16
 * doubles passed to the kernels by value.
 *
 * pred fp32 [h][w] (the frame's depth a), ref_depth fp32 [h][w] (the model's z-depth at ref_pose, no surface unless
 * finite and > 0), ref_normals fp32 [3][h][w] (depth_normals of ref_depth with axes (1, 1, 1): n = 2 c - 1 in the
 * reference camera frame, unusable unless all three are finite).  init_nodes fp64 [2] on the device, the initial (s, t),
 * exactly when affine = 1; with affine = 0, s = 1 and t = 0 are fixed.  With M = ref_pose^-1 T = [Rm tm], a frame pixel
 * with finite a and z = s a + t > 0 has P = z r; Q = Rm P + tm must have Q.z > 0 and its nearest reference pixel q
 * (floor(u + 0.5), floor(v + 0.5)) must lie in the image with a surface and a usable normal n; with V = ref_depth_q r_q,
 * the pair is a correspondence when |Q - V| <= max_dist.  Residual e = n.(Q - V), Huber weight w = min(1, robust / |e|),
 * Jacobian row (m, P x m, m.(a r), m.r) with m = Rm^T n for the step T <- T exp(xi) in the camera frame (the last two
 * entries with affine only).  The normal matrix is scaled to a unit diagonal and solved by Cholesky in fp64.
 * At most `iterations` (1..100) launches; a frame stops when |omega|, |v|, |ds|, |dt| <= tol.  Status (record[1]): 0 ok;
 * 1 no_overlap (fewer than min_overlap, in (0, 1], of the valid pixels have a correspondence); 2 degenerate (a scaled
 * Cholesky pivot below 1e-6, or a zero diagonal); 3 nonfinite (NaN in init_nodes, the sums or the update).  A failed
 * frame returns init_pose and init_nodes (bit for bit).
 *
 * Outputs on the device: pose fp64 [16] (row-major camera-to-world), nodes fp64 [2] (s, t; SparseDepthAligner's
 * grid (1, 1) layout), record fp64 [ODB_TRACK_RECORD] = (correspondences of the last iteration, status, weighted RMS of
 * e in metres, fraction with w < 1, iterations run, s, t, valid frame pixels).  workspace: odb_track_workspace_bytes(h,
 * w) bytes, 8-byte aligned (negative: refused).  A call is a memset of the ticket and iterations + 2 launches, with no
 * host synchronisation, so it can be captured in a CUDA graph.  Fixed pixel chunks and fixed-order sums, no
 * floating-point atomics: results are bit-reproducible.  Arguments are checked before any launch. */
#define ODB_TRACK_RECORD 8
int64_t odb_track_workspace_bytes(int32_t h, int32_t w);
int odb_track_frame(const float* pred, const float* ref_depth, const float* ref_normals, int32_t h, int32_t w,
                    double fx, double fy, double cx, double cy, const double* ref_pose, const double* init_pose,
                    const double* init_nodes, int32_t affine, int32_t iterations, double tol, double robust,
                    double max_dist, double min_overlap, void* workspace, double* pose, double* nodes, double* record,
                    void* stream);

/* odb_track_frame_rgbd: odb_track_frame with a photometric term (DESIGN.md §3 "Camera tracking", photometric term;
 * oracle/photometric_oracle.py restates it in float64).
 * rgb fp32 [3][h][w] is the frame's image and ref_rgb fp32 [3][h][w] the model's colour at ref_pose (NaN: none), both
 * in [0, 1]; ref_intensity fp32 [3][h][w] is scratch the call overwrites with the reference's (Y, g_u, g_v).
 * photometric = lambda finite > 0 (m^2 per squared intensity step), photometric_robust = delta_c finite > 0.
 * Luminance Y = (0.299 R + 0.587 G) + 0.114 B.  A reference pixel is usable with a surface, a finite colour and a usable
 * normal; its gradient (g_u, g_v) is the 3 x 3 Sobel kernel / 8, defined when all 9 window pixels lie in the image, are
 * usable and differ in depth from the centre by at most 5 % of the centre's depth.  Each correspondence of the
 * geometric term whose unrounded projection (u, v) has its bilinear base (floor u, floor v) in [0, w - 2] x [0, h - 2],
 * with finite Y and gradient at the four corners and a finite frame luminance, adds a term: Y, g_u, g_v interpolated x
 * first, e_c = Y_ref(u, v) - Y_frame(p), w_c = min(1, delta_c / |e_c|), the row (m_c, P x m_c, m_c.(a r), m_c.r) with
 * m_c = Rm^T g3, g3 = (g_u fx / Q.z, g_v fy / Q.z, -(g_u fx Q.x + g_v fy Q.y) / Q.z^2), weighted by lambda w_c.  Stopping,
 * statuses and min_overlap (geometric correspondences) are odb_track_frame's.  record fp64 [ODB_TRACK_RGBD_RECORD]:
 * columns 0..7 as odb_track_frame's, then (photometric terms of the last iteration, weighted RMS of e_c, fraction with
 * w_c < 1).  One launch more than odb_track_frame (the reference gradient), same workspace. */
#define ODB_TRACK_RGBD_RECORD 11
int odb_track_frame_rgbd(const float* pred, const float* rgb, const float* ref_depth, const float* ref_rgb,
                         const float* ref_normals, float* ref_intensity, int32_t h, int32_t w, double fx, double fy,
                         double cx, double cy, const double* ref_pose, const double* init_pose,
                         const double* init_nodes, int32_t affine, int32_t iterations, double tol, double robust,
                         double max_dist, double min_overlap, double photometric, double photometric_robust,
                         void* workspace, double* pose, double* nodes, double* record, void* stream);

/* odb_track_information: info fp64 [unknowns][unknowns] (unknowns 6, or 8 with affine) = the normal matrix
 * sum w J J^T of the last Gauss-Newton step that ran in the last odb_track_frame / odb_track_frame_rgbd call on this
 * workspace at h x w (the photometric terms included), unscaled, in the (v, omega[, s, t]) increment coordinates: the
 * per-chunk partials that step left in the workspace, folded in the same order as the step folded them.  Meaningful
 * when that call's status is ok.  One launch; the tracking entry points are unchanged by it. */
int odb_track_information(const void* workspace, int32_t h, int32_t w, int32_t unknowns, double* info, void* stream);

/* ---- SE(3) pose graphs (omnidata_b200/posegraph.py PoseGraph) -----------------------------------------------------
 *
 * No reference counterpart.  Gauss-Newton over N camera-to-world poses T_k with E relative-pose edges (i, j),
 * measurement Z_ij ~ T_i^-1 T_j and information W_ij; node 0 is fixed.  Definition in DESIGN.md §3 "Loop closure and
 * pose graphs"; oracle/posegraph_oracle.py restates it in float64.  All inputs are DEVICE arrays: edges int32 [E][2]
 * (0 <= i, j < N, i != j; the kernels ignore any other edge), poses fp64 [N][16] and measurements fp64 [E][16]
 * (row-major 4 x 4, rigid), information fp64 [E][36] (symmetric).  2 <= N <= ODB_POSEGRAPH_MAX_NODES, 1 <= E <= 8 N.
 *
 * Residual r = Log(Z^-1 T_i^-1 T_j) in (v, omega) order, explicit round-to-nearest fp64: with M = Z^-1 T_i^-1 T_j,
 * w = vee(R_M - R_M^T) / 2, theta = atan2(|w|, (tr R_M - 1) / 2), omega = (theta / |w|) w, v = V^-1 t_M with V^-1 = I -
 * W / 2 + ((1 - A / (2 B)) / theta^2) W^2, W = [omega]x, A = sin(theta) / theta, B = (1 - cos(theta)) / theta^2; below
 * theta = 1e-2 the series theta / |w| = 1 + theta^2 / 6 + 7 theta^4 / 360 and 1 / 12 + theta^2 / 720 + theta^4 / 30240.
 * Increments T_k <- T_k exp(delta_k) (odb_track_frame's exponential); Jacobians d r / d delta_j = I and d r / d delta_i =
 * -Ad(T_j^-1 T_i), Ad(T) = [[R, [t]x R], [0, R]] (Gauss-Newton with J_r^-1(r) ~ I).  H = S J^T W J and g = S J^T W r
 * over the 6 (N - 1) free unknowns, scaled to a unit diagonal, solved by a blocked Cholesky in fp64; a solve stops when
 * every node has |delta_v| <= tol and |delta_omega| <= tol (tol finite > 0), after at most iterations (1..100).
 * Status (record[0]): 0 ok; 1 degenerate (a diagonal entry <= 0, as for a node no edge reaches, or a scaled pivot below
 * 1e-12); 2 nonfinite (a NaN or infinity, or a residual rotation above pi / 2).  A failed solve returns the input poses
 * bit for bit.  poses_out fp64 [N][16]; record fp64 [ODB_POSEGRAPH_RECORD] = (status, iterations run, S r^T W r at the
 * input poses, the same at poses_out, the largest |delta| of the last step, N, E).
 *
 * workspace: odb_posegraph_workspace_bytes(N, E) bytes, 8-byte aligned (negative: refused); it holds the dense fp64
 * matrix, 8 (6 (N - 1))^2 bytes.  A call is 2 + iterations (4 P + 2) launches, P = ceil(6 (N - 1) / 64), with no host
 * synchronisation, so it can be captured in a CUDA graph.  Fixed-order sums, no floating-point atomics: results are
 * bit-reproducible.  Arguments are checked before any launch. */
#define ODB_POSEGRAPH_MAX_NODES 1024
#define ODB_POSEGRAPH_RECORD 7
int64_t odb_posegraph_workspace_bytes(int32_t n_nodes, int32_t n_edges);
int odb_posegraph_optimize(int32_t n_nodes, int32_t n_edges, const int32_t* edges, const double* poses,
                           const double* measurements, const double* information, int32_t iterations, double tol,
                           void* workspace, double* poses_out, double* record, void* stream);

/* ---- place recognition by randomized ferns (omnidata_b200/places.py FernDatabase) ---------------------------------
 *
 * No reference counterpart.  Glocker et al., "Real-time RGB-D camera relocalization via randomized ferns" (2015), as
 * ElasticFusion uses it.  Definition in DESIGN.md §3 "Place recognition and relocalisation"; oracle/places_oracle.py
 * restates it in float64.  All arrays are DEVICE arrays.
 *
 * odb_fern_encode: codes uint8 [n][F] of n frames, depth fp32 [n][h][w] (metres or a relative prediction) and rgb fp32
 * [n][3][h][w]; 1 <= n <= 65535, ODB_FERN_GRID_ROWS <= h <= 65535, ODB_FERN_GRID_COLS <= w <= 65535,
 * 1 <= F <= ODB_FERN_MAX_FERNS.
 *   Thumbnail: cell (r, c) of the 60 x 80 grid covers rows floor(r h / 60) .. floor((r + 1) h / 60) - 1 and columns
 *   floor(c w / 80) .. floor((c + 1) w / 80) - 1.  Each channel (depth, R, G, B) of a cell is the mean of its usable
 *   samples (finite; depth also > 0): summed in fp64 with round-to-nearest adds, rows top to bottom and columns left to
 *   right, divided by the count in fp64 and rounded to fp32; NaN without a usable sample.
 *   Normalisation per frame and channel: m = the lower median (rank floor((n_f - 1) / 2)) of the n_f non-NaN cells,
 *   s = the lower median of |v - m| over them, the difference an fp32 round-to-nearest subtraction.
 *   Ferns: fern f has a cell p_f (fern_cells int32 [F]) and thresholds theta_f,c (fern_thresholds fp64 [F][4]).  Bit c
 *   of code f is (double(v_c(p_f)) - double(m_c)) > theta_f,c double(s_c), both operations round-to-nearest fp64; a
 *   NaN cell, a channel without non-NaN cells or with s = 0, and a cell index outside [0, 4800) give 0.
 *   workspace: odb_fern_encode_workspace_bytes(n) bytes, 8-byte aligned.  3 launches.
 *
 * odb_fern_query: the k entries i < limit of db_codes uint8 [n_db][F] with the smallest distance to code uint8 [F],
 * the distance being the number of ferns whose codes differ; ties to the lower index.  out_index and out_distance
 * int32 [k], in (distance, index) order, padded with -1 beyond min(k, limit).  1 <= n_db <= ODB_FERN_MAX_ENTRIES,
 * 0 <= limit <= n_db,
 * 1 <= k <= ODB_FERN_MAX_K.  workspace: odb_fern_query_workspace_bytes(n_db) bytes, 8-byte aligned.  2 launches.
 *
 * Both only enqueue a fixed launch sequence (no host synchronisation), so they can be captured in a CUDA graph.
 * Integer histograms and scans, no floating-point atomics: outputs are bit-reproducible.  Arguments are checked before
 * any launch. */
#define ODB_FERN_GRID_ROWS 60
#define ODB_FERN_GRID_COLS 80
#define ODB_FERN_MAX_FERNS 4096
#define ODB_FERN_MAX_K 1024
#define ODB_FERN_MAX_ENTRIES (1 << 28)
int64_t odb_fern_encode_workspace_bytes(int32_t n);
int odb_fern_encode(int32_t n, int32_t h, int32_t w, const float* depth, const float* rgb, int32_t n_ferns,
                    const int32_t* fern_cells, const double* fern_thresholds, uint8_t* codes, void* workspace,
                    void* stream);
int64_t odb_fern_query_workspace_bytes(int32_t n_db);
int odb_fern_query(int32_t n_db, int32_t n_ferns, const uint8_t* db_codes, const uint8_t* code, int32_t limit,
                   int32_t k, int32_t* out_index, int32_t* out_distance, void* workspace, void* stream);

/* ---- depth-boundary errors (omnidata_b200/metrics.py BoundaryMetrics) ---------------------------------------------
 *
 * The depth-boundary error (DBE) of iBims-1 (Koch et al., ECCV Workshops 2018): how far predicted depth edges lie from
 * the true ones.  Definitions in DESIGN.md §3 "Depth-boundary metrics"; oracle/boundary_oracle.py restates them in
 * float64.  Inputs fp32 [b][h][w]; mask as for the metrics above; b, h, w <= 65535.  Every value is fp64 with explicit
 * round-to-nearest operations; no floating-point atomics, so results are independent of the batch and
 * bit-reproducible.  workspace: odb_boundary_workspace_bytes(b, h, w) bytes, 8-byte aligned (negative: refused): 31
 * bytes per pixel and 8 * 8 * (slabs + 3) bytes per image, slabs = ceil(h w / 4096).  Arguments are checked before any
 * launch.
 *
 * Edge detector E(f, V), modelled on skimage.feature.canny.  V = {mask != 0, g finite, min_depth < g <= max_depth}
 * (g: the ground truth, or the depth itself for odb_depth_edges); 0 < sigma <= 4, 0 <= low <= high (finite),
 * 0 <= min_depth < max_depth (+inf: none).
 *  1. lo, hi = min, max of f over V.  No edges if |V| = 0, hi = lo or f is not finite somewhere on V; otherwise
 *     fhat = (f - lo) / (hi - lo) on V, 0 elsewhere.
 *  2. Taps w_k = exp(-k^2 / (2 sigma^2)) / S_j exp(-j^2 / (2 sigma^2)), |k| <= R = floor(4 sigma + 0.5), fp64 on the
 *     host.  num = G * (fhat 1_V), den = G * 1_V, separable: along rows, then columns, each a sum over k = -R .. R in
 *     order of w_k v (zeros outside the image); s = num / den where den > 0, else 0.
 *  3. gx = (dx_-1 + 2 dx_0) + dx_1 with dx_j = s[y+j][x+1] - s[y+j][x-1]; gy = (dy_-1 + 2 dy_0) + dy_1 with
 *     dy_j = s[y+1][x+j] - s[y-1][x+j]; m = sqrt(gx^2 + gy^2); m = 0 on the image's one-pixel border.
 *  4. Candidates: the 3x3 neighbourhood lies in the image and in V, m > 0.  With sx, sy = sign(gx), sign(gy) (+1 for
 *     0): if |gx| >= |gy|, w = |gy| / |gx| and the two points interpolate m(x +- sx, y) (1 - w) + m(x +- sx, y +- sy) w;
 *     otherwise w = |gx| / |gy| and m(x, y +- sy) (1 - w) + m(x +- sx, y +- sy) w.  Kept if m >= both.
 *  5. Weak: kept and m >= low; strong: weak and m >= high.  E = the weak pixels whose 8-connected component of weak
 *     pixels holds a strong pixel.
 *
 * odb_depth_edges: edges uint8 [b][h][w] = E(depth, V) (1 = edge).  Eight launches.
 * odb_edge_hysteresis: step 5 alone on weak_strong uint8 [b][h][w] (bit 0 weak, bit 1 strong; a strong pixel counts as
 * weak): edges uint8 [b][h][w].  Four launches.
 * odb_edge_distance2: dist2 uint64 [b][h][w] = the exact squared Euclidean distance in pixels to the nearest edge
 * pixel (nonzero byte) of the image, 0 on one; UINT64_MAX everywhere in an image without edges.  Two launches.
 * odb_boundary_metrics_update: E_p = E(pred, V); E_g = gt_edges (uint8 [b][h][w], nonzero = edge) or, when NULL,
 * E(gt, V).  D_g, D_p = the Euclidean distance transforms of E_g, E_p (sqrt, correctly rounded, of the exact squared
 * distance).  An image with |E_g| = 0 is excluded.  Otherwise A = {p in E_p : D_g(p) < max_dist} (max_dist finite > 0);
 * accuracy = S_A D_g / |A| and completeness = S_{E_g} D_p / |E_g|, both = max_dist when A is empty.  A non-finite pred
 * on V makes them NaN.  records fp64 [b][ODB_BOUNDARY_RECORD] = (accuracy, completeness, |E_p|, |E_g|, |A|, non-finite
 * predictions on V, |E_g| = 0, A empty), NaN errors for an excluded image; state_sums fp64 [2] += (accuracy,
 * completeness) of the images not excluded and state_counts int64 [5] += (1, |E_g| = 0, A empty, |E_p|, |E_g|), image
 * after image in image order.  21 launches (13 with gt_edges).  After a call, the first 8 b h w bytes of the workspace
 * hold D_g^2 as odb_edge_distance2 writes it. */
#define ODB_BOUNDARY_RECORD 8
int64_t odb_boundary_workspace_bytes(int32_t b, int32_t h, int32_t w);
int odb_depth_edges(const float* depth, const void* mask, int32_t mask_dtype, int32_t b, int32_t h, int32_t w,
                    double sigma, double low, double high, double min_depth, double max_depth, void* workspace,
                    uint8_t* edges, void* stream);
int odb_edge_hysteresis(const uint8_t* weak_strong, int32_t b, int32_t h, int32_t w, void* workspace, uint8_t* edges,
                        void* stream);
int odb_edge_distance2(const uint8_t* edges, int32_t b, int32_t h, int32_t w, void* workspace, uint64_t* dist2,
                       void* stream);
int odb_boundary_metrics_update(const float* pred, const float* gt, const void* mask, int32_t mask_dtype,
                                const uint8_t* gt_edges, int32_t b, int32_t h, int32_t w, double sigma, double low,
                                double high, double max_dist, double min_depth, double max_depth, void* workspace,
                                double* records, double* state_sums, int64_t* state_counts, void* stream);

/* ---- test-time ensembles of depth and normal predictions (omnidata_b200/ensemble.py EnsemblePredictor) -----------
 *
 * No reference counterpart: the reference predicts once per image.  Definitions in DESIGN.md §3 "Test-time
 * ensembles"; oracle/ensemble_oracle.py restates them in float64.  members fp32 [k][b][c][h][w]: k predictions of the
 * same b images at h x w, member j stored mirrored (columns reversed) where bit j of `flips` is set; the kernels read
 * them un-mirrored (column w - 1 - x for x).  Member 0 is the reference frame and is never mirrored (bit 0 clear).
 * 1 <= k <= ODB_ENSEMBLE_MAX_MEMBERS, b, h, w <= 65535.  No floating-point atomics: results are independent of the
 * batch and bit-reproducible.  Arguments are checked before any launch.
 *
 * odb_ensemble_gram (depth, c = 1): gram fp64 [b][(k + 1)(k + 2) / 2] = the packed upper triangle (row-major, i <= j)
 * of the Gram matrix of v = (a_0, ..., a_{k-1}, 1) summed over V, the pixels where all k members are finite: entry
 * (j, k) is S a_j, entry (k, k) is n = |V|.  Fixed 4 096-pixel slabs (the partition depends on h x w only), fp64 sums
 * of exact fp32 products, slabs combined in a fixed order.  workspace: odb_ensemble_gram_workspace_bytes(k, b, h, w)
 * bytes, 8-byte aligned (negative: refused).  Two launches.
 * odb_ensemble_align_solve (depth): scale_shift fp64 [b][k][2] = (s_j, t_j) minimising, with s_0 = 1, t_0 = 0,
 *   E = sum_{i<j} sum_{p in V} (s_i a_ip + t_i - s_j a_jp - t_j)^2 + 1e-6 n sum_{j>=1} ((s_j - 1)^2 + t_j^2)
 * from gram: the 2 (k - 1) normal equations by a dense fp64 Cholesky, one CTA per image; k = 1 writes (1, 0).
 * odb_ensemble_merge_depth: per pixel where all members are finite, d_j = fp32(s_j a_j + t_j) (fp64 multiply and add,
 * each rounded to nearest, one rounding to fp32); out fp32 [b][h][w] = the median of the d_j (the middle value for odd
 * k, the fp32 mean (lo + hi) * 0.5 of the two middle values for even k); spread fp32 [b][h][w] (NULL: not written) =
 * the same median of |d_j - out| (fp32).  Elsewhere out = member 0 and spread = NaN.  Not clamped.
 * odb_ensemble_merge_normal (c = 3, the model's encoding [0, 1]): n_j = 2 clamp(a_j, 0, 1) - 1 (a NaN component clamps
 * to 0), the x component (channel 0) negated for a mirrored member; m = (S_j n_j) / k; out fp32 [b][3][h][w] =
 * (m / |m| + 1) / 2, fp64 with round-to-nearest operations and one rounding to fp32, or member 0's clamped value where
 * |m| <= 1e-6; spread fp32 [b][h][w] (NULL: not written) = the mean over j of atan2(|n_j x o|, n_j . o) in degrees,
 * o = 2 out - 1.  The merges read and write 16 bytes per access where w % 4 == 0 and the buffers are 16-byte aligned. */
#define ODB_ENSEMBLE_MAX_MEMBERS 16
int64_t odb_ensemble_gram_workspace_bytes(int32_t k, int32_t b, int32_t h, int32_t w);
int odb_ensemble_gram(const float* members, int32_t k, int32_t flips, int32_t b, int32_t h, int32_t w,
                      void* workspace, double* gram, void* stream);
int odb_ensemble_align_solve(const double* gram, int32_t k, int32_t b, double* scale_shift, void* stream);
int odb_ensemble_merge_depth(const float* members, const double* scale_shift, int32_t k, int32_t flips, int32_t b,
                             int32_t h, int32_t w, float* out, float* spread, void* stream);
int odb_ensemble_merge_normal(const float* members, int32_t k, int32_t flips, int32_t b, int32_t h, int32_t w,
                              float* out, float* spread, void* stream);

/* ---- guided upsampling of a low-resolution prediction (omnidata_b200/guided.py GuidedPredictor) ---------------------
 *
 * No reference counterpart.  The fast guided filter (He & Sun, "Fast Guided Image Filtering", 2015): a local linear
 * model q = a^T I + b of the prediction against the RGB guide, fitted at low resolution and applied to the
 * full-resolution image.  Definitions in DESIGN.md §3 "Guided upsampling"; oracle/guided_oracle.py restates them in
 * float64.  c = 1 (depth) or 3 (normals); b, h, w, H, W <= 65535.  No floating-point atomics: results are independent
 * of the batch and bit-reproducible.  NaN and inf reach every output whose windows or taps touch them.  Arguments are
 * checked before any launch.
 *
 * odb_guided_coefficients: guide fp32 [b][3][h][w], pred fp32 [b][c][h][w].  Window W_i = the pixels within Chebyshev
 * distance radius of i, clipped at the border (1 <= radius <= ODB_GUIDED_MAX_RADIUS); mean_W(f)_i = (S_{W_i} f) / |W_i|,
 * summed down each column, then along the row, in fp64.  mu = mean_W(g), Sigma = mean_W(g g^T) - mu mu^T, m_c =
 * mean_W(p_c), v_c = mean_W(g p_c) - mu m_c; a_c = (Sigma + eps I)^-1 v_c (3x3 Cholesky, eps finite > 0), b_c = m_c -
 * a_c^T mu; coef fp32 [b][4c][h][w]: plane 4 j + k = mean_W(a_jk) (k < 3) and mean_W(b_j) (k = 3), each rounded to fp32
 * once.  workspace: odb_guided_workspace_bytes(b, c, h, w) bytes, 8-byte aligned (negative: refused).  Four launches.
 * odb_guided_apply: out fp32 [b][c][H][W] = B_j + A_j0 x_0 + A_j1 x_1 + A_j2 x_2 (fp32 FMAs in channel order, starting
 * from B_j), image x fp32 [b][3][H][W], where A, B are coef resampled to H x W exactly as odb_resize_bilinear_f32 does
 * with the same tables (bounds_h / weights_h / ksize_h over w -> W, bounds_v / weights_v / ksize_v over h -> H, from
 * omnidata_b200/imageproc.py bilinear_aa_weights).  The resampled coefficients are not written to memory.  16-byte
 * accesses of image and out where W % 4 == 0 and both are 16-byte aligned.  One launch. */
#define ODB_GUIDED_MAX_RADIUS 32
int64_t odb_guided_workspace_bytes(int32_t b, int32_t c, int32_t h, int32_t w);
int odb_guided_coefficients(const float* guide, const float* pred, int32_t b, int32_t c, int32_t h, int32_t w,
                            int32_t radius, double eps, void* workspace, float* coef, void* stream);
int odb_guided_apply(const float* image, const float* coef, int32_t b, int32_t c, int32_t h, int32_t w, int32_t H,
                     int32_t W, const int32_t* bounds_h, const float* weights_h, int32_t ksize_h,
                     const int32_t* bounds_v, const float* weights_v, int32_t ksize_v, float* out, void* stream);

/* ---- Mesh metrics (omnidata_b200/mesh.py, omnidata_b200/metrics.py MeshMetrics) -----------------------------------
 *
 * No reference counterpart.  Measures a reconstructed mesh against a ground-truth mesh: both are sampled the same way,
 * optionally culled to what the cameras saw, and compared by exact nearest neighbours.  Definitions in DESIGN.md §3
 * "Mesh metrics"; oracle/mesh_oracle.py restates them in float64.  Point sets are fp32 [n][3] with n <=
 * ODB_MESH_MAX_POINTS; every fp64 step below is one round-to-nearest operation in the stated order.
 *
 * odb_mesh_sample_count + odb_mesh_sample_emit: vertices fp32 [nv][3], faces int32 [nf][3], density rho finite > 0
 * (points per m^2).  Draws u(t, j) = (x >> 11) 2^-53 with x = splitmix64(splitmix64(key ^ t) ^ j), key =
 * splitmix64(splitmix64(seed) ^ rng_stream).  Face t = (a, b, c): A = 0.5 |(b - a) x (c - a)|, n_t = floor(A rho +
 * u(t, 0)).  Sample k of face t: r1 = u(t, 2k + 1), r2 = u(t, 2k + 2), s = sqrt(r1), p = ((1 - s) a + (s (1 - r2)) b)
 * + (s r2) c, rounded to fp32; samples are ordered by (face, k).  count: writes info int64 [2] = (total, flags) on the
 * device; flags bit 0: a face index outside [0, nv), bit 1: a non-finite vertex used by a face (such faces count 0);
 * workspace odb_mesh_sample_workspace_bytes(nf), 8-byte aligned.  emit: after count on the same workspace, out fp32
 * [total][3]; the caller reads info and refuses flagged meshes and totals above ODB_MESH_MAX_POINTS before emitting.
 *
 * odb_nn_bounds + odb_nn_build + odb_nn_query: for each query q of query fp32 [m][3], distance fp64 [m] = sqrt(d2) and
 * index int32 [m] = the smallest reference index at the minimal d2 = (dx dx + dy dy) + dz dz, dx = (double) q.x -
 * (double) r.x; +inf and -1 when n_ref = 0.  bounds: box int32 [7] = the reference set's order-preserving min keys
 * (x, y, z), max keys, and flags (bit 0: a non-finite reference coordinate, bit 1: a non-finite query coordinate); a
 * float x has the key bits(x) when bits(x) >= 0 as int32, else bits(x) ^ 0x7FFFFFFF.  grid: a HOST array of 7 doubles
 * (lo x, y, z, hi x, y, z, h): finite, lo <= hi, h > 0, n_a = floor((hi_a - lo_a) / h) + 1 cells per axis and at most
 * ODB_NN_MAX_CELLS cells.  A point's cell along axis a is clamp(floor((p_a - lo_a) / h), 0, n_a - 1), for reference
 * points and queries alike.  build: workspace odb_nn_workspace_bytes(n_ref, grid), 16-byte aligned; query: after build
 * on the same workspace and grid.  The cell size changes the time, never an output bit.
 *
 * odb_frustum_mask: mask uint8 [n] = 1 when one of the frames sees the point: cam_to_world a DEVICE array fp64
 * [frames][16] of row-major camera-to-world matrices (checked by the caller), Xc = R^T (X - t), 0 < z <= max_depth and
 * the pixel (floor(fx x / z + cx + 0.5), floor(fy y / z + cy + 0.5)) in the h x w image (odb_tsdf_integrate's
 * projection).  odb_compact_points: out fp32 [count][3] = the points with mask != 0 in order, count int64 [1] on the
 * device; workspace odb_compact_workspace_bytes(n), 8-byte aligned.
 *
 * odb_mesh_metrics_update: one scene from dist_pred fp64 [n_pred] (prediction samples to the ground truth) and dist_gt
 * fp64 [n_gt] (ground truth to the prediction), thresholds a HOST array of 1..ODB_MESH_MAX_THRESHOLDS finite values >
 * 0.  Sums over fixed slabs of 4096 distances, combined in a fixed order; counts of d < t exact.  record fp64
 * [ODB_MESH_RECORD] = (n_pred, n_gt, accuracy, completion, chamfer, then (precision, recall, F) per threshold), NaN
 * where undefined; accuracy = mean dist_pred, completion = mean dist_gt, chamfer = (accuracy + completion) / 2,
 * precision = #(dist_pred < t) / n_pred (0 when n_pred = 0), recall = #(dist_gt < t) / n_gt, F = (2 P R) / (P + R), 0
 * when P + R = 0.  The state: state_counts int64 [7] += (1, n_gt = 0, n_pred = 0 < n_gt, n_pred, n_gt, pred_culled,
 * gt_culled); with n_gt > 0, state_sums fp64 [3 + 3 ODB_MESH_MAX_THRESHOLDS] += (P, R, F) per threshold at [3 + 3k..],
 * and with n_pred > 0 also (accuracy, completion, chamfer) at [0..2].  Workspace
 * odb_mesh_metrics_workspace_bytes(n_pred, n_gt), 8-byte aligned.
 *
 * No floating-point atomics; integer atomics only in the box, the grid's counts, the scatter (no output depends on
 * the order within a cell) and the flags.  Every output is bit-reproducible. */
#define ODB_MESH_MAX_POINTS 268435456
#define ODB_NN_MAX_CELLS 67108864
#define ODB_MESH_MAX_THRESHOLDS 4
#define ODB_MESH_RECORD 17
int64_t odb_mesh_sample_workspace_bytes(int64_t faces);
int odb_mesh_sample_count(const float* vertices, int64_t nv, const int32_t* faces, int64_t nf, double density,
                          int64_t seed, int64_t rng_stream, void* workspace, int64_t* info, void* stream);
int odb_mesh_sample_emit(const float* vertices, int64_t nv, const int32_t* faces, int64_t nf, int64_t seed,
                         int64_t rng_stream, const void* workspace, int64_t total, float* out, void* stream);
int odb_nn_bounds(const float* reference, int64_t n_ref, const float* query, int64_t n_query, int32_t* box,
                  void* stream);
int64_t odb_nn_workspace_bytes(int64_t n_ref, const double* grid);
int odb_nn_build(const float* reference, int64_t n_ref, const double* grid, void* workspace, void* stream);
int odb_nn_query(const float* query, int64_t n_query, int64_t n_ref, const double* grid, const void* workspace,
                 double* distance, int32_t* index, void* stream);
int odb_frustum_mask(const float* points, int64_t n, const double* cam_to_world, int32_t frames, int32_t h, int32_t w,
                     double fx, double fy, double cx, double cy, double max_depth, uint8_t* mask, void* stream);
int64_t odb_compact_workspace_bytes(int64_t n);
int odb_compact_points(const float* points, const uint8_t* mask, int64_t n, void* workspace, float* out,
                       int64_t* count, void* stream);
int64_t odb_mesh_metrics_workspace_bytes(int64_t n_pred, int64_t n_gt);
int odb_mesh_metrics_update(const double* dist_pred, int64_t n_pred, const double* dist_gt, int64_t n_gt,
                            const double* thresholds, int32_t n_thresholds, int64_t pred_culled, int64_t gt_culled,
                            void* workspace, double* record, double* state_sums, int64_t* state_counts,
                            void* stream);

/* Introspection (no GPU needed). */
int odb_abi_version(void);
const char* odb_last_error(void);
/* Number of kernels this library has launched since load (bench.py's gpu_launches). */
int64_t odb_launch_count(void);
/* Diagnostics: when set to a device buffer of grid x (return value) uint64 slots, every following
 * odb_conv_gemm launch stamps %globaltimer at its pipeline events (prologue done, dependency wait done,
 * kernel end; per tile: MMA start / first stage full / MMA commit / epilogue start / epilogue end).
 * NULL switches it off.  Used by profiles/trace_gemm.py; never set on the product path. */
int odb_debug_conv_trace(void* device_buffer);

#ifdef __cplusplus
}
#endif
#endif /* OMNIDATA_B200_H_ */
