// Declarations of the non-GEMM kernels' host launchers (norm.cu, attention.cu, elementwise.cu).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <initializer_list>

namespace t2v {

struct GnShard;      // shard.cuh: cross-rank part of a 5-D GroupNorm of a frame-sharded clip

// ---------------------------------------------------------------- norm.cu
size_t gn_workspace_bytes(int rows_per_inst, int n_inst, int num_sms);
// 0, or -1 (and the reason in t2v_last_error) for arguments groupnorm_silu refuses before touching the workspace
int groupnorm_check(const __half* x, long long ldx, const __half* y, long long ldy, long long rows, int C, int rows_per_inst,
                    const __half* gamma, const __half* beta);
// where the workspace holds the per-(instance, group) (mean, rstd), fp32 [n_inst, 32, 2]: written by phase 1, read by phase 2
float2* gn_workspace_stats(void* workspace);
int groupnorm_silu(const __half* x, long long ldx, __half* y, long long ldy, long long rows, int C, int rows_per_inst,
                   const __half* gamma, const __half* beta, float eps, int silu, void* workspace, int num_sms,
                   cudaStream_t stream, int phase = 0,    // phase 0: stats + apply, 1: stats only, 2: apply only
                   const GnShard* shard = nullptr);       // non-null: statistics are summed over the ranks of a sharded clip
int layernorm(const __half* x, long long ldx, __half* y, long long ldy, long long rows, int C, const __half* gamma,
              const __half* beta, float eps, cudaStream_t stream);

// (mean, rstd) of every row of x over C (LayerNorm statistics; the normalisation itself is folded into the consuming GEMM)
int layernorm_rowstats(const __half* x, long long ldx, long long rows, int C, float eps, float2* out, cudaStream_t stream);

// ---------------------------------------------------------------- attention.cu
struct AttnParams {
    const __half* q;
    const __half* k;
    const __half* v;
    __half* o;
    long long q_bs, q_ss;     // batch / sequence strides in elements (head h lives at column h*head_dim)
    long long k_bs, k_ss;
    long long v_bs, v_ss;
    long long o_bs, o_ss;
    int batch, heads, sq, skv, head_dim;
    int kv_batch_div;         // K/V batch index = q batch index / kv_batch_div (cross-attention: frames share a prompt)
    int b_inner;              // two-level batch: index b -> (b / b_inner) * X_bs + (b % b_inner) * X_bsi
    long long q_bsi, k_bsi, v_bsi, o_bsi;   // (temporal attention: outer = sample, inner = pixel); b_inner = 1 -> unused
    float scale;
};
// Picks the kernel for every caller: attention_tc when attention_tc_eligible (head_dim 64, long sequences), else the
// warp-MMA kernels of attention.cu for head_dim 8 / 16 / 32 / 40 / 64 / 80 / 160 (head h at column h*head_dim).
// Returns -1 without launching on bad shapes, an unsupported head_dim, or operands that break
// attention_operands_aligned's rules on the warp-MMA route.
int attention(const AttnParams& p, cudaStream_t stream);
// What the warp-MMA and relative-position kernels need of their operands: 16-byte cp.async loads (every pointer in
// `loads` 16-byte aligned, every stride in `load_strides` a multiple of 8 elements; 0 is a legal broadcast) and __half2
// stores (O 4-byte aligned, even `o_strides`).  Records the reason with set_error, prefixed by `who`, when it returns false.
bool attention_operands_aligned(const char* who, std::initializer_list<const void*> loads,
                                std::initializer_list<long long> load_strides, const void* o,
                                std::initializer_list<long long> o_strides);

// attention_relpos.cu: temporal attention with relative-position tables (VideoCrafter)
struct RelposParams {
    const __half* q;
    const __half* k;
    const __half* v;
    __half* o;
    const __half* table_k;    // [2*max_rel+1, head_dim] relative_position_k.embeddings_table
    const __half* table_v;    // [2*max_rel+1, head_dim]
    long long n_seq;          // sequences (= samples * pixels); sequence s -> (s / seq_inner, s % seq_inner)
    long long seq_inner;
    long long bs_outer, bs_inner, ss;          // q/k/v: outer / inner sequence strides and the frame stride (elements)
    long long o_bs_outer, o_bs_inner, o_ss;
    int heads, head_dim, T, max_rel;
    float scale;
};
// -1 without launching on bad shapes or on operands that break attention_operands_aligned's rules (the tables are loads too)
int attention_relpos(const RelposParams& p, cudaStream_t stream);

// attention_tc.cu: wgmma / TMA kernel for long self-attention sequences (sq >= 256, skv >= 128, one-level batch).
// attention_tc encodes the three tensor maps before each launch (a captured graph replays them); -1 unless eligible.
bool attention_tc_eligible(const AttnParams& p);
int attention_tc(const AttnParams& p, cudaStream_t stream);

// clip.cu: causal self-attention of the CLIP / OpenCLIP text towers on nn.MultiheadAttention's fused in_proj output
// qkv [B*L, 3W] (q | k | v, head h at columns h*64 of each part) -> o [B*L, W]; q scaled by 64^-0.5 before q.k.
// -1 unless W % 64 == 0, W / heads == 64 and 1 <= L <= 128 (what t2v_clip_create accepts).
int clip_attention(const __half* qkv, __half* o, int B, int L, int W, int heads, cudaStream_t stream);

// ---------------------------------------------------------------- elementwise.cu
// x [B, C, F, h, w] (fp32 or fp16, NCFHW as the samplers hold it) -> tokens [B*F*h*w, ld] fp16, channels >= C zeroed up to cpad
int ingest_latent(const void* x, int x_is_f32, __half* tok, long long ld, int cpad, int B, int C, int F, int h, int w,
                  float scale, cudaStream_t stream);
// the same for frames [frame0, frame0 + nframes) of x in (b f) order (a range may cross a sample boundary; B is implied):
// tokens [nframes*h*w, ld], read straight from the strided latent
int ingest_latent_frames(const void* x, int x_is_f32, __half* tok, long long ld, int cpad, int C, int F, int h, int w,
                         long long frame0, long long nframes, float scale, cudaStream_t stream);
// tokens [B*F*h*w, ld] -> out [B, C, F, h, w] (fp32 or fp16)
int egress_latent(const __half* tok, long long ld, void* out, int out_is_f32, int B, int C, int F, int h, int w,
                  cudaStream_t stream);
int upsample2x(const __half* x, __half* y, int nframes, int h, int w, int C, cudaStream_t stream);
// 3x3 stride-2 pad-1 gather: x [n, h, w, C] -> col [n*ho*wo, 9*C] (tap-major, tap = ky*3+kx)
int im2col_s2(const __half* x, __half* col, int nframes, int h, int w, int C, cudaStream_t stream, int pad_lo = 1);
// T2I-Adapter glue (adapter.cu, unet.cu).  nn.PixelUnshuffle(8): x [N, Cc, H, W] (fp32 or fp16, H, W multiples of 8) ->
// tokens [N*(H/8)*(W/8), 64*Cc] fp16, column c*64 + i*8 + j = x[n, c, 8y+i, 8x+j]
int pixel_unshuffle_ingest(const void* x, int x_is_f32, __half* tok, int N, int Cc, int H, int W, cudaStream_t stream);
// max(x, 0) in place on a dense token matrix [rows, C]; NaN propagates (nn.ReLU)
int relu_inplace(__half* x, long long rows, int C, cudaStream_t stream);
// nn.AvgPool2d(2, 2) (floor sizes): x [n, h, w, C] -> y [n, h/2, w/2, C]; fp32 sum, one fp16 rounding
int avgpool2x2(const __half* x, __half* y, int nframes, int h, int w, int C, cudaStream_t stream);
// x[r, :] += f[(sample % f_samples) * rows_per_sample + r % rows_per_sample, :], sample = r / rows_per_sample; f dense [., C];
// fp16 + fp16 in fp32, one rounding (adding zeros leaves every value unchanged)
int feature_add(__half* x, long long ldx, const __half* f, int C, long long rows, long long rows_per_sample, int f_samples,
                cudaStream_t stream);
int concat_cols(const __half* a, long long lda, int Ca, const __half* b, long long ldb, int Cb, __half* out,
                long long ldo, long long rows, cudaStream_t stream);
// sinusoidal_embedding(t, dim): out [B, dim] fp16 = [cos(t*f_i) | sin(t*f_i)], f_i = 10000^(-i/half)
int time_sinusoid(const float* t, __half* out, int B, int dim, cudaStream_t stream);
// y[b, n] = sum_k act(x[b, k]) * W[n, k] + bias[n] (+ addend[n]) ; act = SiLU if silu_in ; tiny-M linear (M = samples)
int small_linear(const __half* x, long long ldx, const __half* W, const __half* bias, const __half* addend, __half* y,
                 long long ldy, int B, int N, int K, int silu_in, cudaStream_t stream);
int softmax_rows(const __half* x, __half* y, long long rows, int cols, float scale, cudaStream_t stream);
// per-batch transpose: x [nb, R, C] -> y [nb, C, R]
int transpose_batched(const __half* x, __half* y, int nb, int R, int C, cudaStream_t stream);
// decoded tokens [n*H*W, ld] (RGB in cols 0..2, [-1,1]) -> uint8 [n, H, W, 3]: clamp(x*0.5+0.5, 0, 1)*255, truncating
int frames_to_u8(const __half* tok, long long ld, uint8_t* out, long long pixels, cudaStream_t stream);
int frames_to_f32_nchw(const __half* tok, long long ld, float* out, int n, int H, int W, cudaStream_t stream);

// weight packing (source fp16 or fp32, PyTorch layouts)
// conv weight [Cout, Cin, taps] (taps = kh*kw or kt) -> dst [taps][n_alloc][k_alloc] fp16, zero padded
int pack_conv_weight(const void* src, int src_is_f32, __half* dst, int Cout, int Cin, int taps, int n_alloc, int k_alloc,
                     cudaStream_t stream);
// GEGLU proj weight [2*H, K] (+bias [2*H]) -> tile-interleaved rows so one BN-wide accumulator tile holds
// BN/2 value columns followed by their BN/2 gate columns
int pack_geglu_weight(const void* w, const void* b, int src_is_f32, __half* wdst, __half* bdst, int H, int K, int bn,
                      cudaStream_t stream);
int convert_to_f16(const void* src, int src_is_f32, __half* dst, long long n, cudaStream_t stream);
// LoRA merge into a weight in its PyTorch layout [out, cols] (cols = in * kernel taps):
//   w[o, j] = fp16(w[o, j] + fp16(fp16(sum_r B[o, r] A[r, j]) * alpha))                                   (temporal_mean = 0)
//   w[o, i, kt] += alpha * mean_j fp16(sum_r B[o, r] A[r, (i * 3 + kt) * 3 + j]), j = 0..2, same roundings   (temporal_mean = 1, cols = in * 3)
int lora_merge_weight(__half* w, const __half* A, const __half* B, int out, int cols, int rank, float alpha, int temporal_mean,
                      cudaStream_t stream);
// VideoCrafter LoRA merge into a weight in its PyTorch layout [out, cols]: up [out, rank], down [rank, cols], both fp16
// (dtype 0) or fp32 (dtype 1):  w[o, j] = fp16(float(w[o, j]) + alpha * sum_r up[o, r] down[r, j]), fp32 throughout, one rounding
int lora_apply_weight(__half* w, const void* up, const void* down, int dtype, int out, int cols, int rank, float alpha,
                      cudaStream_t stream);
// LayerNorm folded into a Linear: wout[n,k] = fp16(w[n,k] * gamma[k]); colsum[n] = sum_k wout[n,k];
// bias32[n] = sum_k w[n,k] * beta[k] (+ bias[n])
int fold_ln_into_linear(const __half* w, const __half* bias, const __half* gamma, const __half* beta, __half* wout,
                        float* colsum, float* bias32, int N, int K, cudaStream_t stream);

// out[r, n] = fp16( sum_s part[s][r][n] + bias[(r / bias_rows) * bias_stride + n] + residual[r, n] )  (split-K fix-up)
int splitk_reduce(const float* part, int splits, long long split_stride, long long rows, int N, const __half* bias,
                  int bias_rows, long long bias_stride, const __half* residual, long long ldr, __half* out, long long ldo,
                  cudaStream_t stream);

// img2vid inpainting latents: out = img * (1 - w[f]) + noise * w[f] in fp64 (the reference blends in numpy float64,
// process_modelscope.py:199-209); img [BC, img_frames (1 or F), hw] fp32, noise / out / mask [BC, F, hw] fp64, w [F] fp64
int latent_blend(const float* img, int img_frames, const double* noise, const double* w, double* out, double* mask, int BC, int F,
                 long long hw, cudaStream_t stream);

// VideoCrafter q_sample and masked-DDIM blend over a fp32 latent of `shape` [B, C, T, h, w], rounded op by op as torch's fp32
// ops (ddpm3d.py:283-286, ddim.py:194-195): known = a[b]*x0 + s[b]*noise; out = known (mask == null) or
// known*mask + (1 - mask)*img.  x0 / noise / mask take element strides per dimension (0 = broadcast); img / out are contiguous
// (out may be img); a / s hold one coefficient per sample.
struct QSampleBlendParams {
    const float* x0;
    const float* noise;
    const float* a;           // sqrt_alphas_cumprod[t_b], [B]
    const float* s;           // sqrt_one_minus_alphas_cumprod[t_b], [B]
    const float* mask;        // null: q_sample
    const float* img;         // null iff mask is null
    float* out;
    int shape[5];
    long long x0_stride[5], noise_stride[5], mask_stride[5];
};
int q_sample_blend(const QSampleBlendParams& p, cudaStream_t stream);

// sampler updates (fp32 latents [B,C,F,h,w]; eps from the UNet in fp16, cond / uncond)
struct DdimStepParams {
    const float* x;           // x_t
    const void* eps_c;        // conditional eps (fp16, or fp32 when eps_is_f32)
    const void* eps_u;        // unconditional eps (null -> no guidance)
    int eps_is_f32;
    float* x_out;             // x_{t-1}
    long long n;              // elements
    long long chan_stride;    // F*h*w  (elements per channel)
    int C;                    // channels
    int guided_channels;      // channels [0, guided_channels) get u + g (c - u); the rest take eps_c (DDIM_Gaussian quirk)
    float g;                  // guidance scale
    int mode;                 // 0: DDIM_Gaussian op order (gaussian_sampler.py:103-105,:201-202,:280-283)
                              //    x0 = a0*x - a1*e ; eps = (a0*x - x0)/a1 ; x' = a2*x0 + a3*eps + a4*noise
                              // 1: ldm DDIM op order (ddim/sampler.py:200-218)
                              //    x0 = (x - a0*e)/a1 ;                      x' = a2*x0 + a3*e   + a4*noise
    float a0, a1, a2, a3, a4;
    const float* noise;       // may be null when a4 == 0
    int cfg_fp16;             // 1: CFG combine rounded to fp16 op by op, as under the reference's autocast
};
// cfg_variant: 0 u + g (c - u) (fp16 rounding when p.cfg_fp16), 1 c + g (c - u), 2 c + g (u - c), both fp32 only.
// x0_out != null (mode 1 only): also stores x0.  Arguments are checked by the caller; -1 for a variant outside 0..2.
int ddim_step(const DdimStepParams& p, int cfg_variant, float* x0_out, cudaStream_t stream);
// DDIM_Gaussian's step (mode 0) with x0 restricted as gaussian_sampler.py:110-120 does, for B samples of p.n / B elements:
// percentile > 0: s[b] = the percentile-quantile of |x0| of sample b (abs_quantile, written to s; x_out holds x0 meanwhile),
// then x0 = min(s', max(-s', x0)) / s', s' = max(s[b], 1); percentile == 0: x0 clamped to [-1, 1] (s, ws unused).
// Arguments are checked by the caller (t2v_ddim_step_threshold).
int ddim_threshold_step(const DdimStepParams& p, int B, float percentile, float* s, void* ws, cudaStream_t stream);

// ---------------------------------------------------------------- quantile.cu
// out[b] = torch.quantile(|x[b * n, (b + 1) * n)|, q) with linear interpolation, exactly; NaN for a sample holding a NaN.
// ws: abs_quantile_workspace(B) bytes, cleared on the stream by every call.  Arguments are checked by the caller.
constexpr long long kQuantileMaxN = 1LL << 24;      // torch.quantile's limit
size_t abs_quantile_workspace(int B);
int abs_quantile(const float* x, int B, long long n, float q, float* out, void* ws, cudaStream_t stream);
// out = sum_i coef[i] * src[i]  (fp32), n_src <= 8  -- UniPC predictor/corrector combinations
int lincomb(float* out, const float* const* src, const float* coef, int n_src, long long n, cudaStream_t stream);
// CFG combine for UniPC: eps = u + g (c - u) in fp16 rounding, then x0 = (x - sigma*eps)/alpha  -> fp32
int cfg_x0(const float* x, const void* eps_c, const void* eps_u, int eps_is_f32, float* x0, long long n, float g,
           float alpha, float sigma, int cfg_fp16, cudaStream_t stream);

// ---------------------------------------------------------------- resize.cu
// PIL's Image.resize((W, H), LANCZOS) of uint8 RGB frames followed by the reference's x / 255 * 2 - 1, bit for bit.
constexpr int kResizeMaxSize = 32768;
// Pillow's tables for in_size -> out_size pixels (in == out: the identity, one tap): *ksize taps per output, bounds [out][2]
// (first input pixel, taps used), coeffs [out][*ksize] int32 with 22 fractional bits.  bounds / coeffs may be null.
// -1 for a size outside [1, kResizeMaxSize].
int resize_table(int in_size, int out_size, int* ksize, int* bounds, int* coeffs);
// src [n, H0, W0, 3] uint8 -> out [n, 3, H, W] fp32 (or fp16 when out_fp16), through tmp [n, H0, W, 3] uint8 when W != W0.
// Arguments are checked by the caller (t2v_frames_resize).
int frames_resize(const uint8_t* src, int n, int H0, int W0, void* out, int H, int W, int out_fp16, uint8_t* tmp,
                  cudaStream_t stream);

}  // namespace t2v
