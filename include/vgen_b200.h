/*
 * vgen_b200 -- C ABI of libvgen_b200.so: hand-written sm_90a kernels for the VGen sampling hot path
 * (DDIM loop -> spatio-temporal UNet forward -> AutoencoderKL decode).
 *
 * The reference (ali-vilab/VGen) is pure PyTorch and has no FFI for this path: every op below replaces
 * a torch/cuDNN/cuBLAS/xformers library call made from a reference nn.Module.  Each entry cites the
 * reference call site it stands in for (paths relative to the reference root).  The Python classes in
 * vgen_b200/ (registered under the reference's MODEL / DIFFUSION / AUTO_ENCODER registry names) are the
 * only callers; they bind this header with ctypes (see INTEGRATION.md).
 *
 * Conventions
 *   - plain C: raw device pointers, sizes and a cudaStream_t passed as void*; no torch types.
 *   - activations are fp16, channels-last ("tokens x channels", NHWC / [f][h][w][c]); weights fp16,
 *     K-major [out][taps*in]; biases / norm affine fp32; all accumulation fp32.
 *   - every function returns 0 on success; otherwise vgen_last_error() describes the failure.
 *   - no hidden synchronisation, no allocation: the caller owns every buffer (incl. workspaces).
 *   - not thread-safe per stream; one process per GPU.
 */
#ifndef VGEN_B200_H_
#define VGEN_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VGEN_B200_ABI_VERSION 2

/* ---- library ---------------------------------------------------------------------------------- */
int vgen_abi_version(void);
const char* vgen_last_error(void);
/* Number of kernels this library has launched in the calling process (bench.py's gpu_launches). */
int64_t vgen_launch_count(void);
/* tap-GEMM implementation: 0 = auto (default: the wgmma kernel whenever the channel count is a multiple of 64, the SIMT
 * kernel otherwise), 1 = SIMT cross-check kernel everywhere (debug). */
int vgen_set_tapgemm_impl(int impl);
/* tap-GEMM N tile: 0 = heuristic (default); 32..256 in steps of 32 = that tile for every fp16 tap-GEMM launch whose
 * epilogue leaves bn at 0, including vgen_linear_gelu_rowbias (debug: tests reach each kernel instantiation with it).
 * A tile the launch cannot use (GEGLU: bn % 64 != 0 or n % bn != 0; GELU / row bias: bn > 224) fails that launch. */
int vgen_set_tapgemm_bn(int bn);

/* ---- tap-GEMM family (wgmma + TMA; tapgemm_sm90.cu) -------------------------------------------- */
typedef struct vgen_epilogue {
  float alpha;              /* accumulator scale (1.0f = none)                                        */
  const float* bias;        /* [n] fp32 or NULL                                                       */
  const void* group_bias;   /* fp16 [groups][n] or NULL: per-frame bias, added after fp16 rounding     */
  int64_t group_bias_ld;    /*   (ResBlock "h + emb_out": tools/modules/unet/util.py:909-919)          */
  int64_t group_bias_div;   /*   row = image_index / group_bias_div (frames per video); 0 or 1 = per image */
  const void* residual;     /* fp16 [rows][n] or NULL: added after fp16 rounding (skip / x_in adds);  */
  int64_t residual_ld;      /*   not with geglu                                                       */
  int geglu;                /* 1: out[rows][n/2] = value * gelu(gate); W rows interleaved per bn block; */
                            /*   bias 16-byte aligned, no residual / group_bias                       */
  int bn;                   /* N tile (32..256, multiple of 32; GEGLU: multiple of 64); 0 = auto       */
  /* LayerNorm folded into the GEMM (vgen_linear only): with w = W * diag(gamma) (rounded to fp16), col_sum[n] =
   * sum_k w[n][k], bias = b + W beta and row_stats[r] = {rstd_r, -mean_r * rstd_r} (vgen_row_stats),
   *   LN(x) W^T + b  =  rstd_r * (x w^T)[r][n] + (-mean_r rstd_r) * col_sum[n] + bias[n]
   * so the normalised activations are never written (nn.LayerNorm -> nn.Linear, util.py:694-704,731-741).
   * Both NULL = off; GEGLU: col_sum is indexed like bias (packed weight rows). */
  const float* row_stats;   /* fp32 [rows][2] or NULL                                                  */
  const float* col_sum;     /* fp32 [n] or NULL                                                        */
} vgen_epilogue;

/* out[m][n] = epi(a[m][:k] . w[n][:k])       -- nn.Linear / 1x1 conv / Conv1d(k=1)
 * replaces: util.py:224-229 (to_q/k/v/out), :711 (GEGLU.proj), :736 (FF out), :338,:353 (proj_in/out),
 *           :1213,:1229 (Conv1d proj), autoencoder.py:344-363 (q/k/v/proj_out 1x1), :305 (nin_shortcut) */
int vgen_linear(const void* a, int64_t m, int64_t k, int64_t lda, const void* w, int64_t n, void* out,
                int64_t ldo, const vgen_epilogue* epi, void* stream);

/* vgen_linear with a K tail (UNetSD_LoRA's runtime LoRA):
 *   out[m][n] = epi(a[m][:k] . w[n][:k] + h[m][:r] . u[n][:r])
 * both products accumulate into the same fp32 accumulator before the epilogue (bias, residual, one fp16 rounding).  h fp16
 * [m][r] (row stride ldh) is the strength-scaled LoRA down projection of a (vgen_lora_down), u fp16 [n][r] the up weights
 * of every set side by side (block-diagonal over the q / k / v row blocks of a fused projection); r a multiple of 64
 * (zero-padded), h / u 16-byte aligned, ldh a multiple of 8.  epi: alpha, bias, residual, bn; no group_bias, GEGLU or
 * folded LayerNorm.  Same kernels as vgen_linear (vgen_set_tapgemm_impl, vgen_set_tapgemm_bn).
 * replaces: to_q(x) + to_q_lora(x) * scale and the same for k, v and out, tools/modules/unet/unet_lora.py:114-131,161-195 */
int vgen_linear_lora(const void* a, int64_t m, int64_t k, int64_t lda, const void* w, int64_t n, const void* h, int64_t r,
                     int64_t ldh, const void* u, void* out, int64_t ldo, const vgen_epilogue* epi, void* stream);
/* LoRA down projection with the per-sample strength folded in (lora.cu):
 *   h[row][j] = fp16(strength[row / rows_per_sample][col_set[j]] * col_scale[j] * (x[row][:k] . d[j][:k]))   j < r
 *   h[row][j] = 0                                                                                            r <= j < r_pad
 * x fp16 [m][k] (row stride ldx), d fp16 [r][k] (the down weights of every set and every projection reading x, stacked),
 * col_set int32 [r] (the set of column j, < nsets), col_scale fp32 [r] (alpha / rank of that set), strength fp32
 * [m / rows_per_sample][nsets], h fp16 [m][ldh].  k a multiple of 8 up to 2560, x / d 16-byte aligned.
 * replaces: to_q_lora.down_linear(x) (and k, v, out), unet_lora.py:114-131 */
int vgen_lora_down(const void* x, int64_t m, int64_t k, int64_t ldx, const void* d, int64_t r, const int32_t* col_set,
                   const float* col_scale, const float* strength, int64_t nsets, int64_t rows_per_sample, void* h,
                   int64_t ldh, int64_t r_pad, void* stream);

/* Adapter down projection (DreamVideo, tools/modules/unet/util.py:499-519):
 *   out[m][j] = fp16(gelu_erf(a[m][:k] . w[j][:k] + bias[j] + row_bias[m / rows_per_group][j]))
 * with the fp32 row bias added to the fp32 accumulator before the activation (it carries the adapter's condition term
 * lambda * down(condition_linear(c)), one row per frame or per video); bias and row_bias may be NULL.  out may be a
 * column slice of a wider buffer (ldo), e.g. the K tail of [attn_out | h] that the fused output / up projection reads.
 * row_bias: fp32, 8-byte aligned, even ld_row_bias >= n.  Same tap-GEMM kernels as vgen_linear (vgen_set_tapgemm_impl). */
int vgen_linear_gelu_rowbias(const void* a, int64_t m, int64_t k, int64_t lda, const void* w, int64_t n, const float* bias,
                             const float* row_bias, int64_t ld_row_bias, int64_t rows_per_group, void* out, int64_t ldo,
                             void* stream);
/* The condition term of every conditioned adapter of a forward in one launch (adapter.cu):
 *   g[r][j] = lam[r / groups_per_lam] * (c[r][:k] . w[j][:k] + v[j])      (lam NULL: lam_scalar)
 * c fp16 [rows][k] (row stride ldc), w fp16 [n][k] = the stacked products down.W * condition_linear.W, v fp32 [n] = the
 * stacked down.W * condition_linear.b, g fp32 [rows][n] (row stride ldg); k % 8 == 0, c / w 16-byte aligned.
 * replaces: "x + condition_lam * self.condition_linear(condition)" ahead of down_linear, util.py:511-514 */
int vgen_adapter_condition(const void* c, int64_t rows, int64_t k, int64_t ldc, const void* w, const float* v, int64_t n,
                           const float* lam, float lam_scalar, int64_t groups_per_lam, float* g, int64_t ldg, void* stream);

/* 3x3 / stride 1 / pad 1 conv on [nimg][h][w][c] fp16; w is [n][9*c] with k = (ky*3+kx)*c + ci.
 * replaces: nn.Conv2d in ResBlock util.py:845-876, Upsample.conv :761, head unet_t2v.py:204-207,
 *           VAE ResnetBlock / Upsample / conv_in / conv_out autoencoder.py:282-300,448-452,603,647 */
int vgen_conv2d_3x3(const void* x, int64_t nimg, int64_t h, int64_t w_, int64_t c, const void* w, int64_t n,
                    void* out, int64_t ldo, const vgen_epilogue* epi, void* stream);

/* Convolution with an arbitrary list of 1..33 (dy, dx) tap offsets on x [nimg][h][w][c] fp16 (zero padding), w fp16
 * [n][ntaps*c] (tap-major K), output grid = input grid.  Output pixel (b, y, x) is written at
 * out + b*h*out_stride_y + y*out_stride_y + x*out_stride_x (element strides), so one output phase of a transposed conv
 * writes its strided sub-grid directly (out_stride_y != w * out_stride_x needs relu = 1).  relu = 1: relu(acc + bias) in
 * fp32, one rounding (bias only in epi).
 * replaces: nn.ConvTranspose2d(c, c, 4, 2, 1) as four 2x2-tap phases and the stride-1 3x3 convs + ReLU of
 *   tools/annotator/sketch/sketch_simplification.py:27-73; CDCM's conv2_1..conv2_4 summed as one 33-tap conv,
 *   pidinet.py:481-488 */
int vgen_conv2d_taps(const void* x, int64_t nimg, int64_t h, int64_t w_, int64_t c, int64_t ntaps, const int32_t* dy,
                     const int32_t* dx, const void* w, int64_t n, void* out, int64_t out_stride_y, int64_t out_stride_x,
                     const vgen_epilogue* epi, int relu, void* stream);
/* temporal (3,1,1) conv, pad (1,0,0), on [f][hw][c] fp16 (one video); w is [n][3*c], k = kt*c + ci.
 * replaces: nn.Conv3d in TemporalConvBlock_v2 util.py:1662-1680 */
int vgen_tconv3(const void* x, int64_t f, int64_t hw, int64_t c, const void* w, int64_t n, void* out,
                int64_t ldo, const vgen_epilogue* epi, void* stream);
/* the same for `batch` videos stored back to back ([batch][f][hw][c]); frames of different videos never mix */
int vgen_tconv3_batch(const void* x, int64_t batch, int64_t f, int64_t hw, int64_t c, const void* w, int64_t n,
                      void* out, int64_t ldo, const vgen_epilogue* epi, void* stream);

/* ---- FP8 (e4m3) linear (tapgemm_fp8_sm90.cu; opt-in, UNet fp8_linear=True) ------------------------------------- */
/* Row quantiser: x fp16 [m][k] (row stride ldx) -> q e4m3 codes [m][k] (row stride ldq, bytes) and fp32 scale[m] =
 * amax_row / 448, q = e4m3_satfinite(x / scale) rounded to nearest even; an all-zero row gets scale 1.
 * k, ldx, ldq multiples of 8; x 16-byte and q 8-byte aligned. */
int vgen_quantize_rows_e4m3(const void* x, int64_t m, int64_t k, int64_t ldx, void* q, int64_t ldq, float* scale,
                            void* stream);
/* out[m][n] = epi(a_scale[m] * w_scale[n] * (a[m][:k] . w[n][:k]))  with e4m3 a (row stride lda bytes) and w [n][k],
 * fp32 accumulation promoted out of the tensor core every 128 K.  epi: alpha, bias, and either a residual or GEGLU (not
 * both; GEGLU needs a 16-byte aligned bias), and bn (64 or 128; 0 = auto) as for vgen_linear; no group_bias / folded
 * LayerNorm.  k and lda multiples of 16, a / w 16-byte aligned.
 * replaces (opt-in, changes the numerics): the transformer projections of vgen_linear, util.py:224-229,338,353,711,736 */
int vgen_linear_fp8(const void* a, const float* a_scale, int64_t m, int64_t k, int64_t lda, const void* w,
                    const float* w_scale, int64_t n, void* out, int64_t ldo, const vgen_epilogue* epi, void* stream);

/* ---- normalisation (norm.cu; HBM-bound, fp32 statistics) ---------------------------------------- */
/* GroupNorm(32 groups) over x[n][p][c] fp16 (statistics per sample n over p*c/32 values), optional
 * SiLU, y fp16.  For the 5-D (all-frames-jointly) norms pass n = batch, p = f*h*w.
 * replaces: nn.GroupNorm(+nn.SiLU) util.py:845-849,867-869,329,1211,1663-1680; autoencoder.py:15-16 */
int64_t vgen_group_norm_workspace_bytes(int64_t n);
int vgen_group_norm(const void* x, void* y, int64_t n, int64_t p, int64_t c, const float* gamma, const float* beta,
                    float eps, int silu, void* workspace, void* stream);
/* LayerNorm over the last dim of x[rows][c] (row strides ldx / ldy).  replaces: nn.LayerNorm util.py:694-696,1429 */
int vgen_layer_norm(const void* x, void* y, int64_t rows, int64_t c, int64_t ldx, int64_t ldy, const float* gamma,
                    const float* beta, float eps, void* stream);

/* Statistics of that LayerNorm only: stats[rows][2] = {rstd, -mean * rstd} fp32 (two-pass mean / variance like
 * vgen_layer_norm; one read of x, 8 bytes written per row) for a GEMM with vgen_epilogue.row_stats.
 * replaces: the statistics half of nn.LayerNorm util.py:694-696 */
int vgen_row_stats(const void* x, int64_t rows, int64_t c, int64_t ldx, float eps, float* stats, void* stream);

/* ---- attention ---------------------------------------------------------------------------------- */
/* softmax(q k^T * scale) v, head_dim 64, no mask (attn_sm90.cu, wgmma flash attention).  q[batch][lq][heads*64]
 * with token stride ldq (so q/k/v may be column slices of one fused projection buffer); k/v have
 * batch / kv_batch_div batches (a context shared by the frames of a video is stored once).
 * replaces: xformers.ops.memory_efficient_attention, util.py:254-259 (spatial self / cross attention) */
int vgen_attention_d64(const void* q, const void* k, const void* v, void* out, int64_t batch, int64_t heads,
                       int64_t lq, int64_t lk, int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo,
                       int64_t kv_batch_div, float scale, void* stream);
/* Single-head attention with head_dim 512 (attn_sm90.cu, wgmma flash attention: the [lq, lk] score matrix
 * never leaves the SM): out[b][i][:] = softmax_j(q[b][i].k[b][j] * scale) v[b][j][:]; q/k/v/out rows of 512 fp16 with
 * row strides ld* (multiples of 8), batches lq*ld / lk*ld apart.
 * replaces: AttnBlock.forward of the SD VAE, autoencoder.py:365-389 (w_ = bmm(q,k) * c**-0.5; softmax; bmm(v, w_)) */
int vgen_attention_d512(const void* q, const void* k, const void* v, void* out, int64_t batch, int64_t lq, int64_t lk,
                        int64_t ldq, int64_t ldk, int64_t ldv, int64_t ldo, float scale, void* stream);
/* Per-pixel attention over any number L of frames (attn_temporal.cu, mma.sync): token t of
 * sequence s lives at q + s*seq_stride + t*tok_stride (+ head*head_dim).  head_dim 64 is the fast path:
 * register-resident for L <= 32, flash-style (K/V streamed in 64-key blocks, online softmax) for L > 32;
 * any other head_dim <= 64 is served by a scalar kernel (the 4- and 8-channel frame transformers).
 * Videos back to back in one launch: sequence s is pixel (s % seqs_per_batch) of video (s / seqs_per_batch), whose
 * base is q + video*batch_stride (seqs_per_batch <= 0: one video, batch strides ignored).
 * replaces: memory_efficient_attention in TemporalTransformer util.py:1258-1261; Attention util.py:1396-1424 */
int vgen_attention_temporal(const void* q, const void* k, const void* v, void* out, int64_t nseq, int64_t heads,
                            int64_t L, int64_t head_dim, int64_t tok_stride, int64_t seq_stride,
                            int64_t tok_stride_o, int64_t seq_stride_o, int64_t seqs_per_batch, int64_t batch_stride,
                            int64_t batch_stride_o, float scale, void* stream);
/* in-place softmax(x * scale) over rows of x[rows][n] fp16 (VAE AttnBlock, autoencoder.py:377-379) */
int vgen_softmax_rows(void* x, int64_t rows, int64_t n, int64_t ld, float scale, void* stream);

/* ---- data movement / pointwise (elementwise.cu) ------------------------------------------------- */
/* x[n][c][p] (fp32 or fp16) -> y[n][p][c_pad] fp16 (extra channels zero): 'b c f h w -> (b f) h w c' */
int vgen_cp_to_pc(const void* x, int x_is_f32, void* y, int64_t n, int64_t c, int64_t p, int64_t c_pad, void* stream);
/* x[n][p][ldx] fp16 (first c channels) -> y[n][c][p] (fp16 or fp32) */
int vgen_pc_to_cp(const void* x, int64_t ldx, void* y, int y_is_f32, int64_t n, int64_t c, int64_t p, void* stream);
/* channels-last im2col with zero padding (optionally SiLU on the gathered input); columns beyond
 * kh*kw*c up to kpad are zero.  Serves stride-2 / tiny-channel convs (Downsample util.py:946, first
 * conv unet_t2v.py:112, I2VGen conditioning convs unet_i2vgen.py:116-132, VAE conv_in) via vgen_linear */
int vgen_im2col(const void* x, void* out, int64_t nimg, int64_t h, int64_t w, int64_t c, int64_t kh, int64_t kw,
                int64_t stride, int64_t pad_t, int64_t pad_l, int64_t ho, int64_t wo, int64_t kpad, int act_silu,
                void* stream);
/* F.interpolate(scale_factor=2, mode='nearest') on [nimg][h][w][c] (util.py:768, autoencoder.py:455) */
int vgen_upsample_nearest2x(const void* x, void* y, int64_t nimg, int64_t h, int64_t w, int64_t c, void* stream);
/* dst[r][0:cols] = src[r][0:cols] with row strides (torch.cat along channels, unet_t2v.py:269) */
int vgen_copy2d(const void* src, int64_t lds, void* dst, int64_t ldd, int64_t rows, int64_t cols, void* stream);
/* op: 0 silu(a), 1 a+b, 2 gelu(a), 3 a*s, 4 a+s*b, 5 relu(a), 6 quick_gelu(a) = a*sigmoid(1.702a)  (fp16, fp32 math;
 * 6 is OpenAI CLIP's activation, open_clip transformer.py QuickGELU) */
int vgen_eltwise(int op, const void* a, const void* b, void* y, int64_t n, float s, void* stream);
/* out = [gelu](silu_in?(a) @ w^T + bias) [+ res] for small m or tiny k (time / fps / context MLPs
 * unet_t2v.py:93-104, ResBlock emb_layers util.py:857-863, TransformerV2 linears util.py:1396-1452) */
int vgen_linear_small(const void* a, int64_t m, int64_t k, int64_t lda, const void* w, const float* bias, int64_t n,
                      const void* res, int64_t ldr, void* out, int64_t ldo, int silu_in, int gelu_out, void* stream);
/* sinusoidal_embedding util.py:178-190: out[b][dim] fp16 = cat[cos, sin](t * 10000^(-i/half)) */
int vgen_sinusoidal_embedding(const float* t, void* out, int64_t b, int64_t dim, void* stream);
/* nn.AdaptiveAvgPool2d on channels-last input, optional SiLU on the input (unet_i2vgen.py:128-129) */
int vgen_adaptive_avgpool(const void* x, void* y, int64_t nimg, int64_t h, int64_t w, int64_t c, int64_t oh, int64_t ow,
                          int silu_in, void* stream);

/* VideoComposer condition stem (cond_stem.cu): y = AdaptiveAvgPool_{oh x ow}(SiLU(conv3x3_pad1(x) + bias)) in one launch,
 * with no full-resolution intermediate.  x [b][cin][f][h][w] (fp32 or fp16, the engines' layout), 1 <= cin <= 4;
 * weight fp32 [cout][cin][3][3], bias fp32 [cout], cout a multiple of 8 and <= 64; y fp16 channels-last
 * [(b f)][oh][ow][cout] (16-byte aligned).  Pooling bins are PyTorch's (start = floor(i*h/oh), end = ceil((i+1)*h/oh));
 * fp32 accumulation, one rounding at the store.
 * replaces: Conv2d -> SiLU -> AdaptiveAvgPool2d, the first three modules of depth / motion / canny / masked / sketch /
 * single_sketch / local_image_embedding, unet_videolcm.py:295-372 (unet_tf2tv.py:292-369), applied at :598-703 (:594-699) */
int vgen_cond_stem(const void* x, int x_is_f32, int64_t b, int64_t cin, int64_t f, int64_t h, int64_t w, const float* weight,
                   const float* bias, int64_t cout, void* y, int64_t oh, int64_t ow, void* stream);

/* ---- DPT neck and head of the MiDaS v3 depth annotator (dpt.cu; tools/annotator/depth/__init__.py:162-293) ------- */
/* Scatter half of a ConvTranspose2d with kernel == stride == s: g [nimg*hp*wp][ldg] fp16 is the vgen_linear product with
 * the weight repacked to rows (ky, kx, co); out[b][y*s+ky][x*s+kx][co] = fp16(g[(b*hp+y)*wp+x][(ky*s+kx)*cout+co] +
 * bias[co]), channels-last [nimg][s*hp][s*wp][cout].  cout, ldg multiples of 8; g / bias / out 16-byte aligned.
 * replaces: nn.ConvTranspose2d(c, c, 4, stride=4) / (c, c, 2, stride=2), depth/__init__.py:202,212 */
int vgen_dpt_tconv_scatter(const void* g, int64_t ldg, const float* bias, void* out, int64_t nimg, int64_t hp, int64_t wp,
                           int64_t s, int64_t cout, void* stream);
/* F.interpolate(scale_factor=2, mode='bilinear', align_corners=True) on [nimg][h][w][c] fp16 -> [nimg][2h][2w][c]
 * (source coordinate dst * (in - 1) / (out - 1) in fp32, as PyTorch computes it); c a multiple of 8.
 * replaces: depth/__init__.py:158 (FusionBlock), :238 (head nn.Upsample) */
int vgen_upsample_bilinear2x_ac(const void* x, void* y, int64_t nimg, int64_t h, int64_t w, int64_t c, void* stream);
/* Head tail: out[r] = relu(sum_k relu(x[r][k]) * w[k] + bias[0]) for rows r of x [rows][ldx] fp16 (the head's conv3x3
 * output with its bias), w fp32 [c], bias fp32 [1] on the device; out fp16 or fp32 [rows] (= [n][1][H][W]).  c, ldx
 * multiples of 8, c <= 1024.  replaces: ReLU -> nn.ConvTranspose2d(32, 1, 1) -> ReLU, depth/__init__.py:240-242 */
int vgen_dpt_head_out(const void* x, int64_t ldx, int64_t rows, int64_t c, const float* w, const float* bias, void* out,
                      int out_is_f32, void* stream);

/* ---- VideoComposer sketch annotators (sketch.cu; tools/annotator/sketch/pidinet.py, sketch_simplification.py) ------ */
/* Depthwise k x k conv (k = 3 or 5, zero padding, no bias) + ReLU on x [nimg][h][w][c] fp16, c a multiple of 64, wgt fp32
 * [k*k][c].  pool = 1: the conv runs on the 2x2 max-pool of x (floored, as nn.MaxPool2d(2)), which is also written to
 * pooled [nimg][h/2][w/2][c]; out is [nimg][h'][w'][c] with (h', w') the conv's grid.
 * replaces: PDCBlock_converted pool -> conv1 -> relu2, pidinet.py:546-550 */
int vgen_dwconv_relu(const void* x, int64_t nimg, int64_t h, int64_t w, int64_t c, int64_t k, const float* wgt, int pool,
                     void* pooled, void* out, void* stream);
/* CSAM followed by MapReduce on x [nimg][h][w][c] fp16 (c a multiple of 8): t = w1 [4][c] . relu(x) + b1 [4] and
 * s = wm [c] . x per pixel into the fp32 workspaces t_ws [nimg*h*w][4] and s_ws [nimg*h*w], then
 * e = sigmoid(conv3x3(t; w2 [4][3][3])) * s + bm[0] -> fp32 e [nimg][h][w].  All weights fp32 on the device.
 * replaces: CSAM + MapReduce, pidinet.py:458-464,499-500 */
int vgen_csam_mapreduce(const void* x, int64_t nimg, int64_t h, int64_t w, int64_t c, const float* w1, const float* b1,
                        const float* w2, const float* wm, const float* bm, float* t_ws, float* s_ws, float* e, void* stream);
/* PiDiNet's output: bilinear resize (align_corners=False) of the four fp32 side maps e_i [nimg][hw[2i]][hw[2i+1]] to
 * H x W, classifier cw [4] + bias cw[4], sigmoid -> out fp16 or fp32 [nimg][1][H][W].  hw is a host array.
 * replaces: pidinet.py:687-704 */
int vgen_pidinet_fuse(const float* e1, const float* e2, const float* e3, const float* e4, const int64_t* hw, int64_t nimg,
                      int64_t H, int64_t W, const float* cw, void* out, int out_is_f32, void* stream);
/* 3x3 conv (zero padding) to one channel + bias + sigmoid: x [nimg][h][w][c] fp16 (c a multiple of 8), wgt fp32 [9][c],
 * bias fp32 [1] -> out fp16 or fp32 [nimg][1][h][w].  replaces: nn.Conv2d(24, 1, 3, 1, 1) + nn.Sigmoid(),
 * sketch_simplification.py:72-73 */
int vgen_conv3x3_to1_sigmoid(const void* x, int64_t nimg, int64_t h, int64_t w, int64_t c, const float* wgt, const float* bias,
                             void* out, int out_is_f32, void* stream);
/* y = fp16((x - mean) / std) for count elements of fp32 or fp16 x.  replaces: sketch_simplification.py:78 */
int vgen_sketch_normalize(const void* x, int x_is_f32, int64_t count, float mean, float std_, void* y, void* stream);

/* ---- DreamVideo's evaluation metric (metric.cu; metric/cal_metric_DreamVideo.py) ------------------------------------ */
/* torchvision Resize(short side, BICUBIC) -> CenterCrop -> ToTensor -> Normalize of n uint8 RGB images src [n][h][w][3],
 * bit-exact with Pillow's 8-bit ImagingResample (libImaging/Resample.c).  The host passes Pillow's fixed-point tables
 * (22 fractional bits) for the crop's columns and rows only: hbounds [cw][2] = (first source column, taps) and hcoef
 * [cw][kh]; vbounds [ch][2] = (first source row, taps) and vcoef [ch][kv] (an axis Pillow leaves alone: one tap of
 * 1 << 22).  tile_rows is the largest number of source rows the vertical windows of 16 consecutive output rows span.
 * out: fp16 channels-last [n][ch][cw][3] (out_f32 = 0, the towers' input) or fp32 [n][3][ch][cw] (out_f32 = 1, what
 * torchvision returns); (u / 255 - mean[c]) / std[c] in IEEE fp32.
 * replaces: clip_preprocess / dino_preprocess (with T.ToPILImage) per frame, cal_metric_DreamVideo.py:70,78,82,89 */
int vgen_resize_bicubic_crop_normalize(const uint8_t* src, int64_t n, int64_t h, int64_t w, const int32_t* hbounds,
                                       const int32_t* hcoef, int64_t kh, const int32_t* vbounds, const int32_t* vcoef,
                                       int64_t kv, int64_t ch, int64_t cw, int64_t tile_rows, const float* mean3,
                                       const float* std3, void* out, int out_f32, void* stream);
/* The four scores of one video from fp32 features: clip_frames [f][e], text [e], clip_targets [t][e], dino_frames [f][d],
 * dino_targets [t][d] (t may be 0).  Rows are L2-normalised (x / max(||x||, 1e-12)); the frame means are not re-normalised.
 * out4 fp32 = {CLIP-T, CLIP-I, DINO-I, temporal consistency}; t = 0 gives CLIP-I = DINO-I = 0, f = 1 a NaN temporal
 * consistency (the mean of an empty tensor).  One block; (3f + 4t + e + d + 1) floats must fit in 48 KB.
 * replaces: cal_metric_DreamVideo.py:65,74,85,94-124 */
int vgen_video_scores(const float* clip_frames, int64_t f, int64_t e, const float* text, const float* clip_targets,
                      int64_t t, const float* dino_frames, const float* dino_targets, int64_t d, float* out4, void* stream);

/* ---- InstructVideo's segmental video reward (reward.cu) ------------------------------------------------------------ */
/* The HPSv2 image tower's input of n selected frames.  Output frame i reads source frame frame_idx[i] = v * frames_per + t
 * at element offset v * s_video + t * s_frame, channel / row / column strides s_c / s_y / s_x (fp32 [b][3][f][h][w] decoder
 * output, fp32 [n][3][h][w], or uint8 RGB [n][h][w][3] with src_u8 = 1).  Per sample: x * 0.5 + 0.5 (fp32) or x / 255
 * (uint8), clamp(0, 1); then a separable resize with host-computed taps (hbounds [ow][2] = (first source column, taps),
 * hcoef fp32 [ow][kh]; vbounds / vcoef the same for rows; source indices past the edge are clamped): F.interpolate's
 * bilinear, align_corners=False, with or without antialias; then (x - mean[c]) / std[c].  tile_rows: the most source
 * rows the vertical windows of 16 consecutive output rows span.
 * out: fp16 channels-last [n][oh][ow][3] (out_f32 = 0, the image tower's input) or fp32 [n][3][oh][ow] (out_f32 = 1).
 * replaces: reward.py:134-165 (decode output -> mul/add/clamp -> Resize(224) -> Normalize -> frame selection) */
int vgen_reward_frames(const void* src, int src_u8, const int32_t* frame_idx, int64_t n, int64_t frames_per,
                       int64_t s_video, int64_t s_frame, int64_t s_c, int64_t s_y, int64_t s_x, int64_t h, int64_t w,
                       const int32_t* hbounds, const float* hcoef, int64_t kh, const int32_t* vbounds, const float* vcoef,
                       int64_t kv, int64_t oh, int64_t ow, int64_t tile_rows, const float* mean3, const float* std3,
                       void* out, int out_f32, void* stream);
/* reward_scores fp32 [b] of b videos from fp32 image_features [b * s][e] (video-major) and text_features [b][e]:
 * mean over the s segments of <img / max(||img||, 1e-12), txt / max(||txt||, 1e-12)>, each term times
 * exp(-|frame_idx[k * s + j] - f / 2| * lambda_tar) when tar != 0 (frame_idx int32 [b * s], may be null without tar).
 * One block per video.  replaces: reward.py:174-192 */
int vgen_segment_reward(const float* image_features, const float* text_features, const int32_t* frame_idx, int64_t b,
                        int64_t s, int64_t e, int64_t f, int tar, float lambda_tar, float* out, void* stream);

/* ---- the VideoComposer canny annotator (canny.cu) ------------------------------------------------------------------ */
/* cv2.Canny edge maps of n frames of c = 1 or 3 channels, h x w, read at element offset i * s_n + ch * s_c + y * s_y +
 * x * s_x: fp32 in [0, 1] (src_u8 = 0; the bytes are convertScaleAbs(x * 255): |.|, round to nearest even, saturate) or
 * uint8 (src_u8 = 1; taken as they are).  Thresholds per frame, from the exact median m of its h * w * c bytes (float64):
 * mode 0 (low, high) as given; mode 1 (1 - 0.33) * m and (1 + 0.33) * m, truncated, high capped at 255; mode 2
 * trunc((1 - rand[i]) * m) and twice that (rand: fp64 [n] on the device).  Then, as cv2.Canny: swapped if low > high,
 * floored; 3x3 Sobel with replicated borders, the channel with the largest |dx| + |dy|, the L1 magnitude,
 * non-maximum suppression, candidates m > low and strong pixels m > high, and hysteresis: a candidate is an edge when it
 * is 8-connected through candidates to a strong pixel (union-find; the launch count does not depend on the image).
 * Workspaces: bytes uint8 [n][c][h][w], hist int32 [n][256] (zeroed by the call), thr int32 [n][2] (receives the integer
 * low, high), cls uint8 [n][h][w], label int32 [n][h][w], keep uint8 [n][h][w].  out: fp32 [n][h][w] of 0.0 / 1.0 (the
 * condition layout [b][1][f][h][w] for n = b * f).
 * replaces: tools/annotator/canny/__init__.py:23-48 (convertScaleAbs, np.median, cv2.Canny per frame on the host) */
int vgen_canny(const void* src, int src_u8, int64_t n, int64_t c, int64_t h, int64_t w, int64_t s_n, int64_t s_c,
               int64_t s_y, int64_t s_x, int mode, const double* rand, double low, double high, uint8_t* bytes,
               int32_t* hist, int32_t* thr, uint8_t* cls, int32_t* label, uint8_t* keep, float* out, void* stream);

/* ---- the VideoComposer colour-palette annotator (palette.cu) ---------------------------------------------------- */
/* Palette.histogram of n frames of 3 channels (RGB), h x w, read at element offset i * s_n + ch * s_c + y * s_y + x * s_x:
 * src_kind 0 fp32 / 2 fp64 in [0, 1] (widened to fp64), 1 uint8 (linearised through lin, fp64 [256], the sRGB
 * linearisation of v * (1 / 255)).  Per pixel: Lab in fp64 as skimage 0.22 rgb2lab (D65, 2-degree observer), the nearest
 * of the npal <= 156 palette entries lab4 (fp64 [npal][4]: L, a, b and |Lab|^2) by -2 x.y + |x|^2 + |y|^2 clipped at 0,
 * first index on ties; counts into the workspace counts (uint32 [n][npal], zeroed by the call).  Then per frame
 * count / (h * w), and when weight (fp64 [npal][npal], row-normalised exp(-lab_dists / 2 sigma^2)) is given, the smoothed
 * histogram weight . hist with values below 1e-5 set to 0.  out: [n][npal], fp64 (out_f64) or fp32.
 * replaces: tools/annotator/histogram/palette.py:68-81 (rgb2lab, euclidean_distances, argmin, bincount on the host) */
int vgen_palette_histogram(const void* src, int src_kind, int64_t n, int64_t h, int64_t w, int64_t s_n, int64_t s_c,
                           int64_t s_y, int64_t s_x, const double* lab4, int64_t npal, const double* lin,
                           const double* weight, uint32_t* counts, void* out, int out_f64, void* stream);
/* Palette.quantize_image: the same nearest-entry pass, writing qrgb[k] (fp64 [npal][3], lab2rgb of each entry) of the
 * chosen entry k to out, fp64 [n][h][w][3].  replaces: tools/annotator/histogram/palette.py:98-103 */
int vgen_palette_quantize(const void* src, int src_kind, int64_t n, int64_t h, int64_t w, int64_t s_n, int64_t s_c,
                          int64_t s_y, int64_t s_x, const double* lab4, int64_t npal, const double* lin,
                          const double* qrgb, double* out, void* stream);

/* DiagonalGaussianDistribution.sample * scale_factor (autoencoder.py:85-90,211-225): moments fp16 [n][p][2*zc]
 * (mean | logvar, channels-last) + fp32 noise [n][zc][p] -> fp32 z [n][zc][p] */
int vgen_vae_sample(const void* moments, const float* noise, float* z, int64_t n, int64_t zc, int64_t p, float scale,
                    void* stream);

/* ---- model-variant prologues (variants.cu; SURVEY.md section 8 row a21) -------------------------- */
/* softmax(q k^T * scale) v for any head_dim <= 256 and ragged (lq, lk); same addressing as
 * vgen_attention_d64.  Serves the 16-token context transformer of UNetSD_HiGen (head_dim 160) and the CLIP towers
 * (77 causal text tokens, head_dim 64; 257 image tokens, head_dim 80).
 * replaces: CrossAttention / memory_efficient_attention inside TextContextCrossTransformerMultiLayer,
 * unet_higen.py:154-172 (BasicTransformerBlock util.py:674-741) */
int vgen_attention_cross_small(const void* q, const void* k, const void* v, void* out, int64_t batch, int64_t heads,
                               int64_t lq, int64_t lk, int64_t head_dim, int64_t ldq, int64_t ldk, int64_t ldv,
                               int64_t ldo, int64_t kv_batch_div, int causal, float scale, void* stream);
/* CLIP conditioning (clip_embedder.py:183-212 on open_clip's CLIP): causal = 1 above is the text tower's attn_mask.
 * out[r][:] = fp16(table[ids[r]][:] + pos[r % L][:]) -- token_embedding(text) + positional_embedding (:190-191) */
int vgen_embed_tokens(const int64_t* ids, const float* table, const float* pos, void* out, int64_t nrows, int64_t L,
                      int64_t W, int64_t vocab, void* stream);
/* The same gather with textual-inversion vectors (tools/modules/embedding_manager.py:76-116): an id >= vocab selects row
 * id - vocab of extra [n_extra][W] fp32; the caller checks 0 <= id < vocab + n_extra (extra may be NULL iff n_extra == 0) */
int vgen_embed_tokens_extra(const int64_t* ids, const float* table, int64_t vocab, const float* extra, int64_t n_extra,
                            const float* pos, void* out, int64_t nrows, int64_t L, int64_t W, void* stream);
/* x[b][i] = fp16(x[b][i] + add[i]), i < n: "x = x + self.positional_embedding" of the vision tower
 * (utils/reward/open_clip/transformer.py VisionTransformer.forward) */
int vgen_add_rows_f32(void* x, const float* add, int64_t batch, int64_t n, void* stream);
/* F.interpolate(x.transpose(1,2), size=lout, mode='linear').transpose(1,2) on x[nseq][lin][c] fp16
 * (motion embedding, unet_higen.py:389-392) */
int vgen_interp_linear_rows(const void* x, void* y, int64_t nseq, int64_t lin, int64_t lout, int64_t c, void* stream);
/* Fourier_filter(x, threshold=1, scale) of unet_sr600.py:30-49 on channels-last x[nimg][h][w][ldx] (first c
 * channels), written to y[nimg][h][w][ldy]: the four centre bins of the shifted spectrum are scaled. */
int vgen_fourier_lowfreq_filter(const void* x, int64_t ldx, void* y, int64_t ldy, int64_t nimg, int64_t h, int64_t w,
                                int64_t c, float scale, void* stream);
/* UpsampleSR600 (util.py:792-804): nearest x2, keeping output rows [row0, row0+rows_out) of the 2h rows */
int vgen_upsample_nearest2x_rows(const void* x, void* y, int64_t nimg, int64_t h, int64_t w, int64_t c, int64_t row0,
                                 int64_t rows_out, void* stream);
/* dst[r][0:cols] = fp16(src[r][0:cols] * s) with row strides ("x[:, :C/2] *= 1.1", unet_sr600.py:272-273,279) */
int vgen_scale_copy2d(const void* src, int64_t lds, void* dst, int64_t ldd, int64_t rows, int64_t cols, float s,
                      void* stream);

/* ---- sampler ------------------------------------------------------------------------------------ */
/* One fused DDIM update (diffusion_ddim.py:157-162 CFG mix, :194-196 v->x0 | :190-192 eps->x0, :230-240):
 *   out = u + g*(y-u) in fp16 (u NULL: out = y); x0; eps; xt <- c4*x0 + c5*eps (+ c6*noise).
 * coef7 = {sqrt_ab[t], sqrt(1-ab[t]), sqrt(1/ab[t]), sqrt(1/ab[t]-1), sqrt(ab_prev), sqrt(1-ab_prev-sigma^2),
 *          sigma*mask} as fp32 (the host keeps the fp64 tables; timestep/index math is bit-exact there).
 * x0_out (may be NULL) receives the predicted x0, the second value ddim_sample returns (:241). */
int vgen_ddim_step(float* xt, const void* y, const void* u, const float* noise, int64_t n, float guide_scale,
                   const float* coef7, int mean_type_v, float* x0_out, void* stream);

/* GaussianDiffusion (diffusion_gauss.py), the SR600 sampler pair -- sampler_gauss.cu.
 * out[b][n_per] = u + guide_scale*(y-u) in fp16 (:206-210) and stats[b][4] = {sum y, sum y^2, sum out, sum out^2}
 * (fp64, zeroed by the call) for the std-ratio rescale of arXiv:2305.08891 (:212-218). */
int vgen_cfg_combine(const void* y, const void* u, void* out, int64_t batch, int64_t n_per, float guide_scale,
                     double* stats, void* stream);
/* x0 prediction (:220-230) from the fp32 latent xt and the fp16 model output `out`.  stats != NULL applies
 * out *= guide_rescale*std(y)/std(out) + (1-guide_rescale) first.  pred_type: 0 x0, 1 eps, 2 v;
 * alpha/sigma are the table entries of the (batch-uniform) timestep. */
int vgen_gauss_x0(const float* xt, const void* out, const double* stats, float guide_rescale, float alpha, float sigma,
                  int pred_type, float* x0, int64_t batch, int64_t n_per, void* stream);
/* out = a0*x0 + a1*x1 + a2*x2 + a3*x3 (fp32; x1..x3 may be NULL; out may alias an input): model-input
 * scaling (:113), DPM-Solver++(2M) SDE update (:124-139), DDIM inversion step (:408-410) */
int vgen_lincomb_f32(float* out, int64_t n, const float* x0, float a0, const float* x1, float a1, const float* x2,
                     float a2, const float* x3, float a3, void* stream);

/* ---- video write-out ----------------------------------------------------------------------------- */
/* utils/video_op.py:180-192 (save_i2vgen_video_safe; same arithmetic in save_t2vhigen_video_safe :276-288 and
 * save_video_local :226-240): out[f][h][w][3] = uint8(trunc(clamp(video[c][f][h][w]*std[c] + mean[c], 0, 1) * 255)),
 * i.e. mul_, add_, clamp_, *255, 'c f h w -> f h w c', numpy astype('uint8') -- bit-exact, on the device, so frames
 * cross PCIe as bytes.  band_count (may be NULL; f entries, zeroed by the call) receives per frame the number of
 * output bytes in [117, 137]: the last-frame anomaly test of :199-201 (ratio > 0.4 drops the frame). */
int vgen_video_to_rgb8(const float* video, int64_t c, int64_t f, int64_t h, int64_t w, const float* mean3,
                       const float* std3, uint8_t* out, unsigned long long* band_count, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VGEN_B200_H_ */
