/* supir_b200 — C ABI of the H100 (sm_90a) backend for SUPIR's EDM sampling hot path.
 *
 * The reference (Fanghua-Yu/SUPIR) has no FFI: its hot path is a tree of torch.nn modules that dispatch to
 * cuDNN/cuBLAS/ATen. This header is the boundary a maintainer binds instead (ctypes stub in INTEGRATION.md): each entry
 * point names the reference call site(s) it replaces. Conventions:
 *   - plain device pointers + sizes, no torch types; the caller (PyTorch host code) owns every buffer;
 *   - activations are channels-last: images [B, H, W, C] ("NHWC"), tokens [B, L, C] — the same memory;
 *   - bf16 storage unless a name says f32; statistics / softmax / accumulation are fp32 (fp64 for GroupNorm sums);
 *   - `stream` is a cudaStream_t passed as void*; every call is asynchronous on that stream and allocates nothing;
 *   - return 0 on success, negative on error; supir_last_error() returns the message (thread-local);
 *   - devices: calls run on the CALLER's current CUDA device (the one the stream belongs to). The intended deployment is one
 *     process per GPU (torchrun); a process that drives several devices is supported in so far as per-device state (SM count,
 *     opt-in shared-memory sizes of the large kernels) is cached per device, but the tuning knobs (supir_set_*) are per process.
 */
#ifndef SUPIR_B200_H
#define SUPIR_B200_H

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------------------------ */
/* library                                                                                                            */
/* ------------------------------------------------------------------------------------------------------------------ */
const char* supir_last_error(void);
int supir_version(void);
/* number of kernels launched by this library since load / since the last reset (bench.py's gpu_launches) */
long long supir_launch_count(void);
void supir_reset_launch_count(void);

/* ------------------------------------------------------------------------------------------------------------------ */
/* K2/K3/K4: Linear, conv1x1, conv3x3 on wgmma tensor cores (gemm.cu)                                                 */
/* ------------------------------------------------------------------------------------------------------------------ */
typedef struct supir_epilogue {
    const float* bias;      /* [N] fp32 or NULL                      (nn.Linear / nn.Conv2d bias)                      */
    const float* rowvec;    /* [nbatch, rowvec_ld] fp32 or NULL: added per batch element                              */
                            /*   (ResBlock "h + emb_out[..., None, None]", openaimodel.py:343-353)                     */
    int rows_per_batch;     /* GEMM mode: rows per batch element for rowvec (conv mode uses the image index)           */
    int rowvec_ld;          /* leading dim of rowvec (0 -> N)                                                          */
    const void* residual;   /* bf16 [M, ldr] or NULL: added after the bf16 rounding of the GEMM result                 */
    long long ldr;
    int act;                /* 0 none; 1 SiLU; 2 GEGLU (accumulator columns in groups of 32 = 16 value | 16 gate,      */
                            /*   output has N/2 columns; attention.py:84-92, exact-erf GELU)                            */
    int out_f32;            /* 1: out is fp32 instead of bf16                                                          */
    /* LayerNorm folded into the GEMM (attention.py:465-486, norm -> Linear): with A the RAW (un-normalised) rows, W the weight  */
    /* with gamma multiplied into its columns, and bias' = W beta + bias,                                                      */
    /*   LN(a) W^T + bias = rstd * (a W'^T) - (mean * rstd) * colsum(W') + bias'                                               */
    /* ln_stats: [M, 2] fp32 (rstd, mean * rstd) per row from supir_layernorm_stats; ln_colsum: [N] fp32. Both or neither.     */
    const float* ln_stats;
    const float* ln_colsum;
} supir_epilogue;

/* out[M, N] = epilogue(A[M, K] @ W[N, K]^T); A, W bf16 row-major with leading dims lda/ldw (elements, multiples of 8).
 * Replaces nn.Linear (attention.py:213-218, 87, 106, 587, 611; openaimodel.py:287-293) and 1x1 nn.Conv2d on NHWC data
 * (openaimodel.py:317; SUPIR_v0.py:48,87; model.py:124-126,164-175; autoencoder.py:297-298). */
int supir_gemm_bf16(const void* A, long long lda, const void* W, long long ldw, void* out, long long ldc, int M, int N,
                    int K, const supir_epilogue* ep, void* stream);

/* 3x3, stride 1, zero pad 1 convolution on NHWC bf16 as an implicit GEMM (TMA performs the im2col and the padding).
 * x: [B, H, W, ldx>=Cin]; Wp: packed weights [Cout, 3, 3, Cin] (= torch weight.permute(0,2,3,1)); out: [B,H,W,ldc].
 * Replaces nn.Conv2d(k=3,p=1) in ResBlock/ZeroSFT/VAE (openaimodel.py:263,300-307; SUPIR_v0.py:79,82-83; model.py:108-117). */
int supir_conv3x3_bf16(const void* x, long long ldx, const void* Wp, void* out, long long ldc, int B, int H, int W,
                       int Cin, int Cout, const supir_epilogue* ep, void* stream);

/* General small-kernel convolution on NHWC bf16 through the same implicit-GEMM kernel (no im2col buffer): kh x kw taps
 * (1..3 each), stride 1 or 2 (TMA element strides gather every second input pixel), arbitrary tap offset = padding, and an
 * optional interleaved output placement. Input pixel of tap (ky, kx) for output (y, x):
 *   (y * stride + ky + off_y, x * stride + kx + off_x), zero outside the image.
 * Output pixel (y, x) of the Hout x Wout grid is written to (y * out_sy + out_oy, x * out_sx + out_ox) of out
 * [B, out_H, out_W, ldc]. Wp: [Cout, kh, kw, Cin]. Uses:
 *   - Downsample, 3x3 stride 2 pad 1 (openaimodel.py:196-210): off -1, Hout = (Hin - 1) / 2 + 1;
 *   - VAE Downsample, pad (0,1,0,1) then 3x3 stride 2 (model.py:81-85): off 0, Hout = (Hin - 2) / 2 + 1;
 *   - Upsample, nearest 2x then 3x3 pad 1 (openaimodel.py:131-151, model.py:64-68) as FOUR 2x2 convolutions on the
 *     low-resolution input, one per output parity (py, px), with the 3x3 weights pre-summed per parity
 *     (2.25x fewer FLOPs, no 4x intermediate): kh = kw = 2, off = (py - 1, px - 1), out_s = 2, out_o = (py, px). */
typedef struct supir_conv_geometry {
    int kh, kw, stride, off_y, off_x;
    int Hout, Wout;
    int out_sy, out_sx, out_oy, out_ox, out_H, out_W;
} supir_conv_geometry;
int supir_conv_geom_bf16(const void* x, long long ldx, const void* Wp, void* out, long long ldc, int B, int Hin, int Win, int Cin,
                         int Cout, const supir_conv_geometry* geom, const supir_epilogue* ep, void* stream);

/* debugging / tuning knob: force the N tile (64/128/256), 0 = heuristic */
int supir_set_gemm_tile_n(int bn);
/* ------------------------------------------------------------------------------------------------------------------ */
/* network entry / exit convolutions with < 8 channels on one side (smallconv.cu)                                     */
/* ------------------------------------------------------------------------------------------------------------------ */
/* 3x3 pad-1 conv, Cin <= 8: x fp32, addressed x[b*sb + c*sc + y*sy + x] (a strided NCHW view, e.g. a tile of a larger
 * image; the tile border is zero padded like tilevae.py's per-tile convs); w fp32 [Cout, Cin, 3, 3]; optional bf16
 * NHWC residual added to the result ("h += guided_hint", SUPIR_v0.py:531); out NHWC bf16 [B, H, W, ldo].
 * Replaces conv_in / input_hint_block (openaimodel.py:704, SUPIR_v0.py:325,482) and VAE conv_in (model.py:512-514,646-648). */
int supir_conv3x3_small_cin(const float* x, long long sb, long long sc, long long sy, const float* w, const float* bias,
                            const void* residual, long long ldr, void* out, long long ldo, int B, int H, int W, int Cin,
                            int Cout, void* stream);
/* im2col for the same layers as a tensor-core GEMM operand: row p of `out` ([B*H*W, ldo >= KP] bf16) receives the 3x3
 * neighbourhood of pixel p, k = ci * 9 + tap (the flattening of a [Cout][Cin][3][3] weight), zero padded to KP columns and
 * at the image border. supir_gemm_bf16 against the [Cout, KP] weight then replaces supir_conv3x3_small_cin for large images. */
int supir_im2col_3x3_small_cin(const float* x, long long sb, long long sc, long long sy, void* out, long long ldo, int B,
                               int H, int W, int Cin, int KP, void* stream);

/* 3x3 pad-1 conv, Cout in {3,4,8}: x NHWC bf16 [B,H,W,ldx]; w fp32 [Cout, 3, 3, Cin]; only the crop window
 * [crop_y0, crop_y0+crop_h) x [crop_x0, crop_x0+crop_w) of the tile is computed and written to
 * out[b*ob + c*oc + (y-crop_y0)*oy + (x-crop_x0)] (fp32, values rounded to bf16 as under autocast).
 * Replaces UNet `out` conv (openaimodel.py:947-953), VAE conv_out (model.py:563-569,694-696) and, for tiles,
 * crop_valid_region + the paste into the result canvas (tilevae.py:556-567, 946). */
int supir_conv3x3_small_cout(const void* x, long long ldx, const float* w, const float* bias, float* out, long long ob,
                             long long oc, long long oy, int B, int H, int W, int Cin, int Cout, int crop_y0, int crop_x0,
                             int crop_h, int crop_w, void* stream);
/* 1x1 conv on contiguous fp32 NCHW with Cin, Cout <= 8; input pre-multiplied by in_scale (decode: 1/scale_factor).
 * Replaces quant_conv / post_quant_conv (sgm/models/autoencoder.py:297-298, 304-316). */
int supir_conv1x1_small_nchw(const float* x, const float* w, const float* bias, float* y, int B, int Cin, int Cout,
                             long long HW, float in_scale, void* stream);

/* ------------------------------------------------------------------------------------------------------------------ */
/* K1/K5/K13: GroupNorm(32 groups) [+SiLU], ZeroSFT tail, LayerNorm, row softmax (norm.cu)                            */
/* ------------------------------------------------------------------------------------------------------------------ */
/* ws[0 : B*groups*2] (fp64) <- per-(image, group) sum and sum of squares of x [B, HW, ldx>=C] bf16; the rest of the
 * caller-provided workspace (size in doubles from supir_groupnorm_stats_workspace) holds per-block partials so that the
 * reduction order is fixed: results are bit-reproducible run to run. Pass `ws` as `sums` to the apply functions. */
long long supir_groupnorm_stats_workspace(int B, int HW, int C, int groups);
int supir_groupnorm_stats(const void* x, long long ldx, int B, int HW, int C, int groups, double* ws, long long ws_doubles,
                          void* stream);
/* sums -> mean, biased variance (fp32), count = HW * C / groups  (tilevae.py:511-521 get_var_mean) */
int supir_groupnorm_finalize(const double* sums, int n, double count, float* mean, float* var, void* stream);
/* tiled VAE: mean = sum_t w_t mean_t, var = sum_t w_t var_t with w = pixels/max/sum (tilevae.py:629-648) */
int supir_groupnorm_merge_tiles(const float* tile_mean, const float* tile_var, const float* weights, int T, int n,
                                float* mean, float* var, void* stream);
/* y = (x - mean) * rsqrt(var + eps) * gamma + beta, optionally followed by SiLU; statistics either from `sums`
 * (fp64, as written by supir_groupnorm_stats) or from explicit mean/var. GroupNorm32 eps 1e-5 (util.py:258-276),
 * Normalize eps 1e-6 (attention.py:122-125, model.py:49-52); custom_group_norm for tiles (tilevae.py:524-553). */
int supir_groupnorm_apply(const void* x, long long ldx, void* y, long long ldy, int B, int HW, int C, int groups,
                          const double* sums, const float* mean, const float* var, const float* gamma, const float* beta,
                          float eps, int silu, void* stream);
/* ZeroSFT tail (SUPIR_v0.py:110-113): out = lerp(h_raw, GN(h) * (gamma + 1) + beta, *control_scale).
 * h [B,HW,C] is cat(h_ori, skip + zero_conv(c)); h_raw equals h on the first C1 channels and `skip_raw` on the rest;
 * gamma_beta [B,HW,2C] holds the zero_mul | zero_add conv outputs; control_scale is a device scalar. */
int supir_zerosft_apply(const void* h, long long ldh, const void* skip_raw, long long lds, int C1, const void* gamma_beta,
                        long long ldgb, void* out, long long ldo, int B, int HW, int C, int groups, const double* sums,
                        const float* gn_weight, const float* gn_bias, float eps, const float* control_scale, void* stream);
/* nn.LayerNorm over the last dim (attention.py:437-439), eps 1e-5; C % 8 == 0, C <= 2048 */
int supir_layernorm_bf16(const void* x, long long ldx, void* y, long long ldy, long long rows, int C, const float* gamma,
                         const float* beta, float eps, void* stream);
/* per-row LayerNorm statistics only: stats[r] = (rstd, mean * rstd), for the GEMM epilogue's folded LayerNorm (one read
 * pass instead of a read + write pass, and no normalised copy of the activations) */
int supir_layernorm_stats(const void* x, long long ldx, long long rows, int C, float eps, float* stats, void* stream);

/* P = softmax(S * scale) row-wise, fp32 -> bf16 (single-head 512-dim VAE attention, model.py:187-189) */
int supir_softmax_rows(const float* S, long long lds, void* P, long long ldp, long long rows, int cols, float scale,
                       void* stream);

/* ------------------------------------------------------------------------------------------------------------------ */
/* K6: attention, head_dim 64 (attention.cu)                                                                          */
/* ------------------------------------------------------------------------------------------------------------------ */
/* out[b, i, h*64:(h+1)*64] = softmax(q_h k_h^T * scale) v_h ; q [B*Lq, ldq], k/v [B*Lk, ldk/ldv], head h at column h*64.
 * Replaces F.scaled_dot_product_attention / xformers in CrossAttention (attention.py:273-277, 357-359) and
 * ZeroCrossAttn (SUPIR_v0.py:146). */
int supir_attention_bf16(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                         void* out, long long ldo, int B, int H, int Lq, int Lk, int head_dim, float scale, void* stream);
/* Single-head attention with a wide head over L tokens per batch element (the SDXL VAE mid-block AttnBlock, head_dim 512:
 * model.py:158-206, 209-262; tilevae.py:292-336; 128 / 256 for reduced-width VAE configurations):
 * out[b, i, 0:head_dim] = softmax(q k^T * scale) v. q/k/v/out: [B*L, ld] bf16, ld >= head_dim. Flash-style (no score matrix
 * in HBM); at head_dim 512 the two halves of the value columns run as separate CTAs. */
int supir_attention_1head_bf16(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv,
                               void* out, long long ldo, int B, int L, int head_dim, float scale, void* stream);
/* tuning knob: how many of every 4 element pairs of the softmax take 2^x from the FMA-pipe polynomial instead of MUFU.EX2
 * (0..4; default 0 = all on MUFU, or the environment variable SUPIR_B200_ATTN_EMU; negative restores the default). */
int supir_set_attention_exp_emulation(int pairs_of_4);
/* tuning knob: how many of every 4 probability pairs are rounded / packed to bf16 with integer instructions on the ALU pipe
 * instead of cvt.rn.bf16x2.f32, which shares the XU pipe with the exponentials (0..4; environment SUPIR_B200_ATTN_ALU_PACK;
 * negative restores the default). */
int supir_set_attention_alu_pack(int pairs_of_4);

/* ------------------------------------------------------------------------------------------------------------------ */
/* K7/K8/K10/K12/K14 and data movement (elementwise.cu)                                                               */
/* ------------------------------------------------------------------------------------------------------------------ */
/* nearest 2x upsample on NHWC bf16 (openaimodel.py:131-151, model.py:64-68) */
int supir_upsample_nearest2x(const void* x, long long ldx, void* y, long long ldy, int B, int H, int W, int C, void* stream);
/* im2col for 3x3 stride-2 convs: out [B*Ho*Wo, 9*C]; pad_lo = 1 (UNet Downsample, openaimodel.py:196-210) or
 * 0 (VAE Downsample pads right/bottom only, model.py:81-85) */
int supir_im2col_3x3_s2(const void* x, long long ldx, void* out, int B, int H, int W, int C, int Ho, int Wo, int pad_lo,
                        void* stream);
int supir_copy2d_bf16(const void* src, long long lds, void* dst, long long ldd, long long rows, int cols, void* stream);
/* out = a + y * (*scale)  (ZeroCrossAttn, SUPIR_v0.py:150) */
int supir_axpy_bf16(const void* a, long long lda, const void* y, long long ldy, void* out, long long ldo, long long rows,
                    int cols, const float* scale, void* stream);
int supir_nchw_f32_to_nhwc_bf16(const float* x, void* y, long long ldy, int B, int C, int HW, void* stream);
int supir_nhwc_bf16_to_nchw_f32(const void* x, long long ldx, float* y, int B, int C, int HW, void* stream);
/* crop window [crop_y0, +crop_h) x [crop_x0, +crop_w) of an NHWC bf16 tile [B, H, W, ldx >= C] -> fp32 NCHW view with element
 * strides (ob, oc, oy, 1): the exit of a network whose last conv ran on the tensor cores with Cout padded to 8 */
int supir_nhwc_bf16_crop_to_nchw_f32(const void* x, long long ldx, float* y, long long ob, long long oc, long long oy, int B,
                                     int H, int W, int C, int crop_y0, int crop_x0, int crop_h, int crop_w, void* stream);
int supir_f32_to_bf16(const float* x, void* y, long long n, void* stream);
/* timestep_embedding (sgm/modules/diffusionmodules/util.py:206-230), dim even, max_period 1e4 */
int supir_timestep_embedding(const float* t, float* out, int B, int dim, void* stream);
/* y = [silu]( [silu](x) @ W^T + bias ) [+ add] for B <= 16 rows (time/label embedding MLPs, per-ResBlock emb_layers:
 * openaimodel.py:664-697, 287-293); x, y, add fp32; W bf16 [N, K]. silu_out bit 0: SiLU before the add; bit 1: SiLU of the
 * final sum (emb is only ever consumed through SiLU -> Linear, so its SiLU is computed once here instead of per consumer) */
int supir_linear_small_m(const float* x, int ldx, const void* W, const float* bias, float* y, int ldy, int B, int N, int K,
                         int silu_in, int silu_out, const float* add, int ldadd, void* stream);
/* sampler step, part 1 (sampling.py:550-556 + guiders.py:65-74 + denoiser.py:71): x_hat = x + eps*noise_mul (eps may be
 * NULL); net_in[0:n] = net_in[n:2n] = x_hat * c_in */
int supir_edm_pre(const float* x, const float* eps, float noise_mul, float c_in, float* x_hat, float* net_in, long long n,
                  void* stream);
/* sampler step, part 2 (denoiser.py:73, guiders.py:59-63, sampling.py:563-569): denoised = net*c_out + x_hat per branch,
 * CFG mix u + s (c - u), optional restore guidance den -= (den - x_center) * restore_mul, Euler update */
int supir_edm_post(const float* x_hat, const float* net_out, const float* x_center, float c_out, float cfg_scale,
                   float restore_mul, float sigma_hat, float dt, float* x_next, float* denoised, long long n, void* stream);
/* unfused sampler arithmetic for callers that keep the reference's denoiser/guider objects in the loop:
 * out = a*alpha + b*beta (b may be NULL; denoiser.py:73, sampling.py:556,567-569) and the CFG pair reduction
 * out[n] = u_n + scale[n] * (c_n - u_n) with x = [u ; c] (guiders.py:59-63, sampling_utils.py:7-9) */
int supir_axpby_f32(const float* a, float alpha, const float* b, float beta, float* out, long long n, void* stream);
int supir_cfg_combine(const float* x, const float* scale, float* out, int N, long long per_sample, void* stream);
/* K12 (sampling.py:629-659): out = (sum_j tiles_j * w) / (sum_j w) over the windows covering each pixel, accumulated in
 * window order with fp64 products rounded to fp32 after every add. tiles [num_windows, N, C, tile, tile] fp32;
 * windows int32 [num_windows, 4] = (hi, hi_end, wi, wi_end), hi < 0 marks an unused slot; weights fp64 [tile, tile].
 * supir_tile_gather is the matching window extraction (sampling.py:633-641): out[j] = src[:, :, window j]. */
int supir_tile_gather(const float* src, const int* windows, int num_windows, int tile, float* out, int N, int C, int H,
                      int W, void* stream);
int supir_tile_blend(const float* tiles, const int* windows, int num_windows, int tile, const double* weights, float* out,
                     int N, int C, int H, int W, void* stream);
/* K14 (distributions.py:24-41, SUPIR_model.py:45,61): z = scale * (mean + exp(0.5*clamp(logvar)) * eps), eps NULL = mode */
int supir_gaussian_latent(const float* moments, const float* eps, float scale, float* z, int B, int Cz, long long HW,
                          void* stream);

/* ------------------------------------------------------------------------------------------------------------------ */
/* text conditioner (textenc.cu; SURVEY.md section 8(f)2): CLIP-L and OpenCLIP bigG text towers, once per image          */
/* ------------------------------------------------------------------------------------------------------------------ */
/* out[r, 0:C] = table[idx[r], 0:C] (+ pos[r % L, 0:C] when pos != NULL), fp32; idx int32, clamped to [0, table_rows).
 * Replaces the nn.Embedding lookups + positional add of the text towers (HF CLIPTextEmbeddings behind
 * sgm/modules/encoders/modules.py:494-496; open_clip token_embedding + positional_embedding, modules.py:569-570) and the
 * EOT-row gather of `pool` (modules.py:584-590: x[arange, text.argmax(-1)]). */
int supir_gather_rows_f32(const float* table, long long ldt, int table_rows, const int* idx, const float* pos, long long ldp,
                          int L, float* out, long long ldo, long long rows, int C, void* stream);
/* nn.LayerNorm over fp32 rows (the towers keep their residual stream in fp32: autocast lowers only the matmuls), written as
 * bf16 (y_bf16, the next GEMM's operand) and / or fp32 (y_f32: ln_final, modules.py:574,580); either may be NULL.
 * Replaces layer_norm1/2 + final_layer_norm of HF CLIPEncoderLayer and ln_1 / ln_2 / ln_final of open_clip's resblocks. */
int supir_layernorm_f32(const float* x, long long ldx, void* y_bf16, long long ldyb, float* y_f32, long long ldyf, long long rows,
                        int C, const float* gamma, const float* beta, float eps, void* stream);
/* softmax(q k^T * scale [+ causal mask]) v for short sequences: L <= 128 tokens, head_dim 64; q/k/v/out bf16 [B*L, ld], head h at
 * column h*64. Replaces the text towers' masked self-attention (HF CLIPAttention with the causal mask; open_clip
 * nn.MultiheadAttention(attn_mask=model.attn_mask), modules.py:571,592-607). */
int supir_attention_small_bf16(const void* q, long long ldq, const void* k, long long ldk, const void* v, long long ldv, void* out,
                               long long ldo, int B, int H, int L, int head_dim, float scale, int causal, void* stream);
/* y = act(x) on bf16 rows (x, y may alias): mode 0 exact GELU (open_clip nn.GELU), mode 1 quick-GELU x * sigmoid(1.702 x)
 * (openai/clip-vit-large-patch14 `hidden_act`). */
int supir_activation_bf16(const void* x, long long ldx, void* y, long long ldy, long long rows, int cols, int mode, void* stream);

/* ------------------------------------------------------------------------------------------------------------------ */
/* colour fix on the decoded image (colorfix.cu; SUPIR/utils/colorfix.py, SURVEY.md section 8(f)1)                     */
/* ------------------------------------------------------------------------------------------------------------------ */
/* one a-trous wavelet level on fp32 NCHW planes: low = blur(img) with the 3x3 kernel [1 2 1]x[1 2 1]/16 at dilation
 * `radius` and replicate padding (wavelet_blur, colorfix.py:73-92); high (+)= img - low (wavelet_decomposition :94-106).
 * high may be NULL; accumulate = 0 overwrites high. img and low must not alias. */
int supir_wavelet_level(const float* img, float* low, float* high, int planes, int H, int W, int radius, int accumulate,
                        void* stream);
/* per-plane (sum, sum of squares) in fp64 -> ws[0 : 2*planes]; deterministic; workspace size from the helper */
long long supir_plane_stats_workspace(int planes);
int supir_plane_stats(const float* x, int planes, long long hw, double* ws, long long ws_doubles, void* stream);
/* adaptive_instance_normalization (colorfix.py:45-71): (content - mean_c) / std_c * std_s + mean_s, unbiased var + 1e-5 */
int supir_adain_apply(const float* content, const double* content_stats, const double* style_stats, float* out, int planes,
                      long long hw, void* stream);
/* Tensor2PIL (SUPIR/util.py:87-94): bicubic resize of one fp32 [C, H, W] image in [-1, 1] to (h0, w0) exactly as
 * torch.nn.functional.interpolate(mode='bicubic') computes it, then * 127.5 + 127.5, clip, truncate: out uint8 [h0, w0, C]. */
int supir_image_to_uint8_bicubic(const float* x, int C, int H, int W, unsigned char* out, int h0, int w0, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SUPIR_B200_H */
