// C-ABI glue: library state + the kernel-level entry points of include/t2v_b200.h.
#include "../../include/t2v_b200.h"
#include "common.cuh"
#include "gemm_tc.cuh"
#include "kernels.cuh"

#include <cstdarg>
#include <cstdio>
#include <cstring>

namespace t2v {

static char g_err[512] = "";
static int g_device = -1;
static int g_num_sms = 132;
static void* g_gn_ws = nullptr;
static size_t g_gn_ws_bytes = 0;

void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}
int num_sms() { return g_num_sms; }
void clear_pending_error(const char* where) {
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess)
        fprintf(stderr, "[t2v_b200] %s: clearing a pending CUDA error left by an earlier call: %s (%s)\n", where, cudaGetErrorString(e),
                cudaGetErrorName(e));
}
int launch_status(const char* what) {
    const cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess) return 0;
    set_error("%s: %s (%s)", what, cudaGetErrorString(e), cudaGetErrorName(e));
    return -2;
}

static void* gn_scratch(size_t bytes) {
    if (bytes > g_gn_ws_bytes) {
        if (g_gn_ws) cudaFree(g_gn_ws);
        g_gn_ws = nullptr;
        if (cudaMalloc(&g_gn_ws, bytes) != cudaSuccess) return nullptr;
        cudaMemset(g_gn_ws, 0, bytes);
        g_gn_ws_bytes = bytes;
    }
    return g_gn_ws;
}

}  // namespace t2v

using namespace t2v;

extern "C" {

int t2v_init(int device) {
    if (cudaSetDevice(device) != cudaSuccess) {
        set_error("cudaSetDevice(%d) failed: %s", device, cudaGetErrorString(cudaGetLastError()));
        return -1;
    }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) {
        set_error("cudaGetDeviceProperties failed");
        return -1;
    }
    if (prop.major != 9 || prop.minor != 0) {
        set_error("t2v_b200 is built for sm_90a only; device %d is sm_%d%d", device, prop.major, prop.minor);
        return -2;
    }
    g_device = device;
    g_num_sms = prop.multiProcessorCount;
    if (gemm_init() != 0) {
        set_error("gemm_init failed (driver entry point / smem attribute)");
        return -3;
    }
    return 0;
}
const char* t2v_last_error(void) { return g_err; }
int t2v_num_sms(void) { return g_num_sms; }
const char* t2v_version(void) { return "t2v_b200 0.2 (sm_90a; wgmma+TMA implicit GEMM)"; }

}  // extern "C"

// the problem of t2v_op_gemm's arguments (also t2v_op_gemm_splitk's)
static GemmProblem op_problem(const void* a, long long lda, int K, int nd, const int* dims, int ntaps, const int* tap_off,
                              const void* w_packed, int n_alloc, int N, int b_batch_dim, int flags, void* out, long long ldo,
                              const void* bias, int bias_rows, long long bias_stride, const void* residual, long long ldr,
                              float alpha, int force_bn, int force_cg) {
    GemmProblem p;
    memset(&p, 0, sizeof(p));
    p.a = reinterpret_cast<const __half*>(a);
    p.lda = lda;
    p.K = K;
    p.nd = nd;
    for (int d = 0; d < nd; ++d) p.dim[d] = dims[d];
    p.ntaps = ntaps;
    for (int t = 0; t < ntaps; ++t)
        for (int d = 0; d < nd; ++d) p.tap_off[t][d] = tap_off ? tap_off[t * nd + d] : 0;
    p.b = reinterpret_cast<const __half*>(w_packed);
    p.n_alloc = n_alloc;
    p.N = N;
    p.b_batch_dim = b_batch_dim;
    p.flags = flags & ~(GEMM_DBG_FORCE_BS | GEMM_DBG_NO_BS | GEMM_DBG_SLAB_OUT);
    p.force_bs = (flags & GEMM_DBG_FORCE_BS) ? 1 : ((flags & GEMM_DBG_NO_BS) ? -1 : 0);
    p.slab_out = (flags & GEMM_DBG_SLAB_OUT) ? 1 : 0;
    p.out = out;
    p.ldo = ldo;
    p.bias = reinterpret_cast<const __half*>(bias);
    p.bias_rows = bias_rows;
    p.bias_stride = bias_stride;
    p.residual = reinterpret_cast<const __half*>(residual);
    p.ldr = ldr;
    p.alpha = alpha;
    p.force_bn = force_bn;
    p.force_cg = force_cg;
    return p;
}

static int plan_op(const GemmProblem& p, GemmPlan* plan, const char* what) {
    const int rc = gemm_plan(p, plan, g_num_sms);
    if (rc != 0) set_error("%s: gemm_plan failed (%d)", what, rc);
    return rc;
}

static int launch_op(const GemmPlan& plan, const char* what, cudaStream_t stream) {
    const int rc = gemm_launch(plan, stream);
    if (rc != 0) set_error("%s: gemm_launch failed: %s", what, cudaGetErrorString(cudaGetLastError()));
    return rc;
}

extern "C" {

int t2v_op_gemm(const void* a, long long lda, int K, int nd, const int* dims, int ntaps, const int* tap_off,
                const void* w_packed, int n_alloc, int N, int b_batch_dim, int flags, void* out, long long ldo,
                const void* bias, int bias_rows, long long bias_stride, const void* residual, long long ldr,
                float alpha, int force_bn, int force_cg, void* stream) {
    const GemmProblem p = op_problem(a, lda, K, nd, dims, ntaps, tap_off, w_packed, n_alloc, N, b_batch_dim, flags, out, ldo, bias,
                                     bias_rows, bias_stride, residual, ldr, alpha, force_bn, force_cg);
    GemmPlan plan;
    const int rc = plan_op(p, &plan, "op_gemm");
    return rc != 0 ? rc : launch_op(plan, "op_gemm", reinterpret_cast<cudaStream_t>(stream));
}

int t2v_op_gemm_splitk(const void* a, long long lda, int K, int nd, const int* dims, int ntaps, const int* tap_off,
                       const void* w_packed, int n_alloc, int N, int b_batch_dim, int flags, void* out, long long ldo,
                       const void* bias, int bias_rows, long long bias_stride, const void* residual, long long ldr,
                       float alpha, int splits, float* scratch, long long scratch_elems, int* splits_used, int force_bn,
                       int force_cg, void* stream) {
    const GemmProblem p = op_problem(a, lda, K, nd, dims, ntaps, tap_off, w_packed, n_alloc, N, b_batch_dim, flags, out, ldo, bias,
                                     bias_rows, bias_stride, residual, ldr, alpha, force_bn, force_cg);
    if (const char* why = gemm_splitk_unsupported(p)) {
        set_error("op_gemm_splitk: split-K does not take this problem: %s", why);
        return -1;
    }
    if (splits < 1 || scratch == nullptr || splits_used == nullptr) {
        set_error("op_gemm_splitk: needs splits >= 1, a scratch buffer and a place for the split count");
        return -1;
    }
    const int S = gemm_split_count(p, splits);
    const long long need = gemm_splitk_scratch_elems(p, S);
    if (scratch_elems < need) {
        set_error("op_gemm_splitk: %d splits need %lld fp32 scratch elements, the buffer holds %lld", S, need, scratch_elems);
        return -1;
    }
    GemmPlan plan;
    int rc = plan_op(gemm_splitk_partials(p, S, scratch), &plan, "op_gemm_splitk");
    if (rc != 0) return rc;
    *splits_used = S;
    const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    rc = launch_op(plan, "op_gemm_splitk", s);
    if (rc != 0) return rc;
    rc = gemm_splitk_reduce(p, S, scratch, s);
    if (rc != 0) set_error("op_gemm_splitk: splitk_reduce failed (%d)", rc);
    return rc;
}

int t2v_op_ln_linear(const void* x, long long ldx, long long rows, int K, const void* w, const void* bias, const void* gamma,
                     const void* beta, int N, int flags, void* w_folded, float* colsum, float* bias32, float* rowstat,
                     const void* residual, long long ldr, void* out, long long ldo, int force_bn, int force_cg, void* stream) {
    if (!x || !w || !gamma || !beta || !w_folded || !colsum || !bias32 || !rowstat || !out) {
        set_error("op_ln_linear: x, w, gamma, beta, out and the four intermediate buffers are required");
        return -1;
    }
    if ((flags & ~GEMM_GEGLU) != 0) {
        set_error("op_ln_linear: flags must be 0 or GEMM_GEGLU (%d)", flags);
        return -1;
    }
    if (K % 8 != 0 || K > 2048 || rows < 1 || rows >= (1LL << 31) || N < 1) {
        set_error("op_ln_linear: LayerNorm rows need K %% 8 == 0 and K <= 2048, 1 <= rows < 2^31 (K %d rows %lld N %d)", K, rows, N);
        return -1;
    }
    // the GEMM of ln_linear (runtime.cu): weights pre-scaled by gamma, out = rstd_r * (acc - mean_r * colsum_n) + bias32_n
    GemmProblem p;
    memset(&p, 0, sizeof(p));
    p.a = reinterpret_cast<const __half*>(x);
    p.lda = ldx;
    p.K = K;
    p.nd = 1;
    p.dim[0] = static_cast<int>(rows);
    p.ntaps = 1;
    p.b = reinterpret_cast<const __half*>(w_folded);
    p.n_alloc = N;
    p.N = N;
    p.b_batch_dim = -1;
    p.flags = flags | GEMM_LN;
    p.out = out;
    p.ldo = ldo;
    p.residual = reinterpret_cast<const __half*>(residual);
    p.ldr = ldr;
    p.alpha = 1.0f;
    p.force_bn = force_bn;
    p.force_cg = force_cg;
    p.rowstat = reinterpret_cast<const float2*>(rowstat);
    p.colsum = colsum;
    p.bias32 = bias32;
    GemmPlan plan;
    int rc = plan_op(p, &plan, "op_ln_linear");
    if (rc != 0) return rc;
    const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    rc = fold_ln_into_linear(reinterpret_cast<const __half*>(w), reinterpret_cast<const __half*>(bias),
                             reinterpret_cast<const __half*>(gamma), reinterpret_cast<const __half*>(beta),
                             reinterpret_cast<__half*>(w_folded), colsum, bias32, N, K, s);
    if (rc == 0) rc = layernorm_rowstats(p.a, ldx, rows, K, 1e-5f, reinterpret_cast<float2*>(rowstat), s);
    if (rc != 0) {
        set_error("op_ln_linear: fold / row statistics launch failed (%d)", rc);
        return rc;
    }
    return launch_op(plan, "op_ln_linear", s);
}

int t2v_latent_blend(const float* image_latents, int image_frames, const double* noise, const double* weights, double* out,
                     double* mask_out, int BC, int F, long long hw, void* stream) {
    if ((image_frames != 1 && image_frames != F) || BC < 1 || F < 1 || hw < 1) {
        set_error("latent_blend: image_frames must be 1 or F");
        return -1;
    }
    return latent_blend(image_latents, image_frames, noise, weights, out, mask_out, BC, F, hw, reinterpret_cast<cudaStream_t>(stream));
}

int t2v_q_sample_blend(const float* x0, const long long* x0_strides, const float* noise, const long long* noise_strides,
                       const float* a, const float* s, const float* mask, const long long* mask_strides, const float* img,
                       float* out, const int* shape, void* stream) {
    if (!x0 || !x0_strides || !noise || !noise_strides || !a || !s || !out || !shape) {
        set_error("q_sample_blend: x0, noise, a, s, out, their strides and the shape are required");
        return -1;
    }
    if ((mask == nullptr) != (img == nullptr) || (mask && !mask_strides)) {
        set_error("q_sample_blend: mask and img go together (both null for q_sample), and a mask needs strides");
        return -1;
    }
    QSampleBlendParams p;
    memset(&p, 0, sizeof(p));
    p.x0 = x0;
    p.noise = noise;
    p.a = a;
    p.s = s;
    p.mask = mask;
    p.img = img;
    p.out = out;
    for (int d = 0; d < 5; ++d) {
        if (shape[d] < 1) {
            set_error("q_sample_blend: shape[%d] = %d, every dimension must be >= 1", d, shape[d]);
            return -1;
        }
        if (x0_strides[d] < 0 || noise_strides[d] < 0 || (mask && mask_strides[d] < 0)) {
            set_error("q_sample_blend: negative stride in dimension %d", d);
            return -1;
        }
        p.shape[d] = shape[d];
        p.x0_stride[d] = x0_strides[d];
        p.noise_stride[d] = noise_strides[d];
        p.mask_stride[d] = mask ? mask_strides[d] : 0;
    }
    return q_sample_blend(p, reinterpret_cast<cudaStream_t>(stream));
}

int t2v_resize_coeffs(int in_size, int out_size, int* ksize, int* bounds, int* coeffs) {
    if (ksize == nullptr || resize_table(in_size, out_size, ksize, bounds, coeffs) != 0) {
        set_error("resize_coeffs: sizes must lie in [1, %d] (in %d, out %d) and ksize must not be null", kResizeMaxSize, in_size,
                  out_size);
        return -1;
    }
    return 0;
}

int t2v_frames_resize(const void* src, int n, int H0, int W0, void* out, int H, int W, int out_fp16, void* tmp,
                      long long tmp_bytes, void* stream) {
    const int M = kResizeMaxSize;
    if (n < 1 || H0 < 1 || W0 < 1 || H < 1 || W < 1 || H0 > M || W0 > M || H > M || W > M) {
        set_error("frames_resize: n must be >= 1 and every size in [1, %d] (n %d, %dx%d -> %dx%d)", M, n, W0, H0, W, H);
        return -1;
    }
    if (src == nullptr || out == nullptr) {
        set_error("frames_resize: src and out are required");
        return -1;
    }
    const size_t esize = out_fp16 ? sizeof(__half) : sizeof(float);
    if (reinterpret_cast<uintptr_t>(out) % esize != 0) {
        set_error("frames_resize: out must be aligned to its element size (%zu bytes)", esize);
        return -1;
    }
    const long long need = W != W0 ? static_cast<long long>(n) * H0 * W * 3 : 0;
    if (W != W0 && (tmp == nullptr || tmp_bytes < need)) {
        set_error("frames_resize: resizing %d to %d columns needs a uint8 buffer of %lld bytes, got %lld", W0, W, need,
                  tmp ? tmp_bytes : 0LL);
        return -1;
    }
    clear_pending_error("frames_resize");
    return frames_resize(static_cast<const uint8_t*>(src), n, H0, W0, out, H, W, out_fp16, static_cast<uint8_t*>(tmp),
                         reinterpret_cast<cudaStream_t>(stream));
}

int t2v_op_pack_conv_weight(const void* src, int src_is_f32, void* dst, int Cout, int Cin, int taps, int n_alloc,
                            int k_alloc, void* stream) {
    return pack_conv_weight(src, src_is_f32, reinterpret_cast<__half*>(dst), Cout, Cin, taps, n_alloc, k_alloc,
                            reinterpret_cast<cudaStream_t>(stream));
}
int t2v_op_lora_merge(void* w, const void* A, const void* B, int out, int cols, int rank, float alpha, int temporal_mean,
                      void* stream) {
    if (rank < 1 || out < 1 || cols < 1) {
        set_error("op_lora_merge: rank, out and cols must be >= 1 (rank %d, out %d, cols %d)", rank, out, cols);
        return -1;
    }
    clear_pending_error("op_lora_merge");
    return lora_merge_weight(reinterpret_cast<__half*>(w), reinterpret_cast<const __half*>(A), reinterpret_cast<const __half*>(B),
                             out, cols, rank, alpha, temporal_mean, reinterpret_cast<cudaStream_t>(stream));
}
int t2v_op_lora_apply(void* w, const void* up, const void* down, int dtype, int out, int cols, int rank, float alpha,
                      void* stream) {
    if (rank < 1 || out < 1 || cols < 1 || (dtype != 0 && dtype != 1)) {
        set_error("op_lora_apply: rank, out and cols must be >= 1 and dtype 0 (fp16) or 1 (fp32) (rank %d, out %d, cols %d, "
                  "dtype %d)", rank, out, cols, dtype);
        return -1;
    }
    clear_pending_error("op_lora_apply");
    return lora_apply_weight(reinterpret_cast<__half*>(w), up, down, dtype, out, cols, rank, alpha,
                             reinterpret_cast<cudaStream_t>(stream));
}
int t2v_op_pack_geglu_weight(const void* w, const void* b, int src_is_f32, void* wdst, void* bdst, int H, int K, int bn,
                             void* stream) {
    return pack_geglu_weight(w, b, src_is_f32, reinterpret_cast<__half*>(wdst), reinterpret_cast<__half*>(bdst), H, K, bn,
                             reinterpret_cast<cudaStream_t>(stream));
}
int t2v_op_groupnorm(const void* x, long long ldx, void* y, long long ldy, long long rows, int C, int rows_per_inst,
                     const void* gamma, const void* beta, float eps, int silu, int phase, float* stats, void* stream) {
    const __half* xh = reinterpret_cast<const __half*>(x);
    __half* yh = reinterpret_cast<__half*>(y);
    const __half* gh = reinterpret_cast<const __half*>(gamma);
    const __half* bh = reinterpret_cast<const __half*>(beta);
    if (phase < 0 || phase > 2 || (phase != 0 && stats == nullptr)) {
        set_error("op_groupnorm: phase %d must be 0, 1 or 2, and phases 1 and 2 need a stats buffer", phase);
        return -1;
    }
    if (groupnorm_check(xh, ldx, yh, ldy, rows, C, rows_per_inst, gh, bh) != 0) return -1;
    const int n_inst = static_cast<int>(rows / rows_per_inst);
    void* ws = gn_scratch(gn_workspace_bytes(rows_per_inst, n_inst, g_num_sms));
    if (!ws) {
        set_error("groupnorm workspace allocation failed");
        return -5;
    }
    const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const size_t stats_bytes = static_cast<size_t>(n_inst) * 32 * sizeof(float2);
    if (phase == 2 && cudaMemcpyAsync(gn_workspace_stats(ws), stats, stats_bytes, cudaMemcpyDeviceToDevice, s) != cudaSuccess)
        return launch_status("op_groupnorm: statistics copy");
    const int rc = groupnorm_silu(xh, ldx, yh, ldy, rows, C, rows_per_inst, gh, bh, eps, silu, ws, g_num_sms, s, phase);
    if (rc != 0 || phase != 1) return rc;
    if (cudaMemcpyAsync(stats, gn_workspace_stats(ws), stats_bytes, cudaMemcpyDeviceToDevice, s) != cudaSuccess)
        return launch_status("op_groupnorm: statistics copy");
    return 0;
}
int t2v_op_layernorm(const void* x, long long ldx, void* y, long long ldy, long long rows, int C, const void* gamma,
                     const void* beta, float eps, void* stream) {
    return layernorm(reinterpret_cast<const __half*>(x), ldx, reinterpret_cast<__half*>(y), ldy, rows, C,
                     reinterpret_cast<const __half*>(gamma), reinterpret_cast<const __half*>(beta), eps,
                     reinterpret_cast<cudaStream_t>(stream));
}
int t2v_op_attention(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_ss,
                     long long k_bs, long long k_ss, long long v_bs, long long v_ss, long long o_bs, long long o_ss,
                     int batch, int heads, int sq, int skv, int kv_batch_div, float scale, void* stream) {
    AttnParams p;
    p.q = reinterpret_cast<const __half*>(q);
    p.k = reinterpret_cast<const __half*>(k);
    p.v = reinterpret_cast<const __half*>(v);
    p.o = reinterpret_cast<__half*>(o);
    p.q_bs = q_bs; p.q_ss = q_ss; p.k_bs = k_bs; p.k_ss = k_ss; p.v_bs = v_bs; p.v_ss = v_ss; p.o_bs = o_bs; p.o_ss = o_ss;
    p.batch = batch; p.heads = heads; p.sq = sq; p.skv = skv; p.head_dim = 64; p.kv_batch_div = kv_batch_div;
    p.scale = scale; p.b_inner = 1; p.q_bsi = p.k_bsi = p.v_bsi = p.o_bsi = 0;
    return attention(p, reinterpret_cast<cudaStream_t>(stream));
}
int t2v_op_attention_hd(const void* q, const void* k, const void* v, void* o, long long q_bs, long long q_ss,
                        long long k_bs, long long k_ss, long long v_bs, long long v_ss, long long o_bs, long long o_ss,
                        int batch, int heads, int head_dim, int sq, int skv, int kv_batch_div, float scale, int b_inner,
                        long long q_bsi, long long k_bsi, long long v_bsi, long long o_bsi, void* stream) {
    AttnParams p;
    memset(&p, 0, sizeof(p));
    p.q = reinterpret_cast<const __half*>(q);
    p.k = reinterpret_cast<const __half*>(k);
    p.v = reinterpret_cast<const __half*>(v);
    p.o = reinterpret_cast<__half*>(o);
    p.q_bs = q_bs; p.q_ss = q_ss; p.k_bs = k_bs; p.k_ss = k_ss; p.v_bs = v_bs; p.v_ss = v_ss; p.o_bs = o_bs; p.o_ss = o_ss;
    p.batch = batch; p.heads = heads; p.sq = sq; p.skv = skv; p.head_dim = head_dim; p.kv_batch_div = kv_batch_div;
    p.scale = scale; p.b_inner = b_inner;
    p.q_bsi = q_bsi; p.k_bsi = k_bsi; p.v_bsi = v_bsi; p.o_bsi = o_bsi;
    return attention(p, reinterpret_cast<cudaStream_t>(stream));
}
int t2v_op_attention_relpos(const void* q, const void* k, const void* v, void* o, const void* table_k, const void* table_v,
                            long long n_seq, long long seq_inner, long long bs_outer, long long bs_inner, long long ss,
                            long long o_bs_outer, long long o_bs_inner, long long o_ss, int heads, int head_dim, int T,
                            int max_rel, float scale, void* stream) {
    RelposParams p;
    memset(&p, 0, sizeof(p));
    p.q = reinterpret_cast<const __half*>(q);
    p.k = reinterpret_cast<const __half*>(k);
    p.v = reinterpret_cast<const __half*>(v);
    p.o = reinterpret_cast<__half*>(o);
    p.table_k = reinterpret_cast<const __half*>(table_k);
    p.table_v = reinterpret_cast<const __half*>(table_v);
    p.n_seq = n_seq; p.seq_inner = seq_inner; p.bs_outer = bs_outer; p.bs_inner = bs_inner; p.ss = ss;
    p.o_bs_outer = o_bs_outer; p.o_bs_inner = o_bs_inner; p.o_ss = o_ss;
    p.heads = heads; p.head_dim = head_dim; p.T = T; p.max_rel = max_rel; p.scale = scale;
    return attention_relpos(p, reinterpret_cast<cudaStream_t>(stream));
}
int t2v_op_upsample2x(const void* x, void* y, int nframes, int h, int w, int C, void* stream) {
    return upsample2x(reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y), nframes, h, w, C,
                      reinterpret_cast<cudaStream_t>(stream));
}
int t2v_op_im2col_s2(const void* x, void* col, int nframes, int h, int w, int C, int pad_lo, void* stream) {
    if (pad_lo != 0 && pad_lo != 1) {
        set_error("op_im2col_s2: pad_lo must be 0 or 1 (got %d)", pad_lo);
        return -1;
    }
    const int rc = im2col_s2(reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(col), nframes, h, w, C,
                             reinterpret_cast<cudaStream_t>(stream), pad_lo);
    if (rc == -1) set_error("op_im2col_s2: C = %d must be a multiple of 8", C);
    return rc;
}
int t2v_op_ingest_latent(const void* x, int x_is_f32, void* tok, long long ld, int cpad, int C, int F, int h, int w,
                         long long frame0, long long nframes, float scale, void* stream) {
    return ingest_latent_frames(x, x_is_f32, reinterpret_cast<__half*>(tok), ld, cpad, C, F, h, w, frame0, nframes, scale,
                                reinterpret_cast<cudaStream_t>(stream));
}
int t2v_op_egress_latent(const void* tok, long long ld, void* out, int out_is_f32, int B, int C, int F, int h, int w,
                         void* stream) {
    return egress_latent(reinterpret_cast<const __half*>(tok), ld, out, out_is_f32, B, C, F, h, w,
                         reinterpret_cast<cudaStream_t>(stream));
}
int t2v_op_avgpool2x2(const void* x, void* y, int nframes, int h, int w, int C, void* stream) {
    const int rc = avgpool2x2(reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y), nframes, h, w, C,
                              reinterpret_cast<cudaStream_t>(stream));
    if (rc == -1) set_error("op_avgpool2x2: C = %d must be a multiple of 8", C);
    return rc;
}
int t2v_op_pixel_unshuffle(const void* x, int x_is_f32, void* tok, int N, int Cc, int H, int W, void* stream) {
    const int rc = pixel_unshuffle_ingest(x, x_is_f32, reinterpret_cast<__half*>(tok), N, Cc, H, W,
                                          reinterpret_cast<cudaStream_t>(stream));
    if (rc == -1) set_error("op_pixel_unshuffle: H = %d and W = %d must be multiples of 8", H, W);
    return rc;
}
int t2v_op_relu(void* x, long long rows, int C, void* stream) {
    const int rc = relu_inplace(reinterpret_cast<__half*>(x), rows, C, reinterpret_cast<cudaStream_t>(stream));
    if (rc == -1) set_error("op_relu: C = %d must be a multiple of 8", C);
    return rc;
}
int t2v_op_feature_add(void* x, long long ldx, const void* f, int C, long long rows, long long rows_per_sample, int f_samples,
                       void* stream) {
    const int rc = feature_add(reinterpret_cast<__half*>(x), ldx, reinterpret_cast<const __half*>(f), C, rows, rows_per_sample,
                               f_samples, reinterpret_cast<cudaStream_t>(stream));
    if (rc == -1)
        set_error("op_feature_add: C = %d and ldx = %lld must be multiples of 8, rows_per_sample = %lld and f_samples = %d >= 1", C,
                  ldx, rows_per_sample, f_samples);
    return rc;
}
int t2v_op_concat_cols(const void* a, long long lda, int Ca, const void* b, long long ldb, int Cb, void* out, long long ldo,
                       long long rows, void* stream) {
    const int rc = concat_cols(reinterpret_cast<const __half*>(a), lda, Ca, reinterpret_cast<const __half*>(b), ldb, Cb,
                               reinterpret_cast<__half*>(out), ldo, rows, reinterpret_cast<cudaStream_t>(stream));
    if (rc == -1)
        set_error("op_concat_cols: Ca = %d, Cb = %d, lda = %lld, ldb = %lld and ldo = %lld must be multiples of 8", Ca, Cb, lda, ldb,
                  ldo);
    return rc;
}
int t2v_op_softmax_rows(const void* x, void* y, long long rows, int cols, float scale, void* stream) {
    return softmax_rows(reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y), rows, cols, scale,
                        reinterpret_cast<cudaStream_t>(stream));
}
int t2v_op_transpose_batched(const void* x, void* y, int nb, int R, int C, void* stream) {
    return transpose_batched(reinterpret_cast<const __half*>(x), reinterpret_cast<__half*>(y), nb, R, C,
                             reinterpret_cast<cudaStream_t>(stream));
}
int t2v_op_frames_to_u8(const void* tok, long long ld, void* out, long long pixels, void* stream) {
    return frames_to_u8(reinterpret_cast<const __half*>(tok), ld, reinterpret_cast<uint8_t*>(out), pixels,
                        reinterpret_cast<cudaStream_t>(stream));
}
int t2v_op_frames_to_f32(const void* tok, long long ld, float* out, int n, int H, int W, void* stream) {
    return frames_to_f32_nchw(reinterpret_cast<const __half*>(tok), ld, out, n, H, W, reinterpret_cast<cudaStream_t>(stream));
}
int t2v_op_convert_to_f16(const void* src, int src_is_f32, void* dst, long long n, void* stream) {
    return convert_to_f16(src, src_is_f32, reinterpret_cast<__half*>(dst), n, reinterpret_cast<cudaStream_t>(stream));
}
int t2v_op_time_sinusoid(const float* t, void* out, int B, int dim, void* stream) {
    return time_sinusoid(t, reinterpret_cast<__half*>(out), B, dim, reinterpret_cast<cudaStream_t>(stream));
}
int t2v_op_small_linear(const void* x, long long ldx, const void* W, const void* bias, const void* addend, void* y,
                        long long ldy, int B, int N, int K, int silu_in, void* stream) {
    return small_linear(reinterpret_cast<const __half*>(x), ldx, reinterpret_cast<const __half*>(W),
                        reinterpret_cast<const __half*>(bias), reinterpret_cast<const __half*>(addend),
                        reinterpret_cast<__half*>(y), ldy, B, N, K, silu_in, reinterpret_cast<cudaStream_t>(stream));
}
int t2v_ddim_step(const float* x, const void* eps_c, const void* eps_u, int eps_is_f32, float* x_out, long long n, long long chan_stride,
                  int C, int guided_channels, float g, int mode, float a0, float a1, float a2, float a3, float a4,
                  const float* noise, int cfg_fp16, void* stream) {
    DdimStepParams p;
    p.x = x; p.eps_c = eps_c; p.eps_u = eps_u; p.eps_is_f32 = eps_is_f32;
    p.x_out = x_out; p.n = n; p.chan_stride = chan_stride; p.C = C; p.guided_channels = guided_channels; p.g = g;
    p.mode = mode; p.a0 = a0; p.a1 = a1; p.a2 = a2; p.a3 = a3; p.a4 = a4; p.noise = noise; p.cfg_fp16 = cfg_fp16;
    return ddim_step(p, 0, nullptr, reinterpret_cast<cudaStream_t>(stream));
}
static bool ranges_overlap(const void* a, long long a_bytes, const void* b, long long b_bytes) {
    if (a == nullptr || b == nullptr) return false;
    const uintptr_t pa = reinterpret_cast<uintptr_t>(a), pb = reinterpret_cast<uintptr_t>(b);
    return pa < pb + static_cast<uintptr_t>(b_bytes) && pb < pa + static_cast<uintptr_t>(a_bytes);
}
int t2v_ddim_step_ex(const float* x, const void* eps_c, const void* eps_u, int eps_is_f32, float* x_out, long long n,
                     long long chan_stride, int C, int guided_channels, float g, int mode, float a0, float a1, float a2, float a3,
                     float a4, const float* noise, int cfg_fp16, int cfg_variant, float* x0_out, void* stream) {
    if (cfg_variant < 0 || cfg_variant > 2) {
        set_error("ddim_step_ex: cfg_variant must be 0 (None), 1 ('cfg_original') or 2 ('cfg_ours'), got %d", cfg_variant);
        return -1;
    }
    if (cfg_variant != 0 && cfg_fp16 != 0) {
        set_error("ddim_step_ex: cfg_variant %d is fp32 only (cfg_fp16 must be 0)", cfg_variant);
        return -1;
    }
    if (x0_out != nullptr) {
        if (mode != 1) {
            set_error("ddim_step_ex: x0_out needs mode 1 (the ldm / VideoCrafter DDIM update), got mode %d", mode);
            return -1;
        }
        const long long f32 = n * 4, eps = n * (eps_is_f32 ? 4 : 2);
        if (ranges_overlap(x0_out, f32, x, f32) || ranges_overlap(x0_out, f32, x_out, f32) ||
            ranges_overlap(x0_out, f32, eps_c, eps) || ranges_overlap(x0_out, f32, eps_u, eps) ||
            ranges_overlap(x0_out, f32, noise, f32)) {
            set_error("ddim_step_ex: x0_out overlaps x, x_out, eps_c, eps_u or noise");
            return -1;
        }
    }
    DdimStepParams p;
    p.x = x; p.eps_c = eps_c; p.eps_u = eps_u; p.eps_is_f32 = eps_is_f32;
    p.x_out = x_out; p.n = n; p.chan_stride = chan_stride; p.C = C; p.guided_channels = guided_channels; p.g = g;
    p.mode = mode; p.a0 = a0; p.a1 = a1; p.a2 = a2; p.a3 = a3; p.a4 = a4; p.noise = noise; p.cfg_fp16 = cfg_fp16;
    clear_pending_error("ddim_step_ex");
    return ddim_step(p, cfg_variant, x0_out, reinterpret_cast<cudaStream_t>(stream));
}
long long t2v_abs_quantile_workspace(int B) { return static_cast<long long>(abs_quantile_workspace(B)); }
static int check_quantile_args(const char* what, const float* x, int B, long long n, const float* out, const void* ws,
                               long long ws_bytes) {
    if (B < 1 || B > 65535 || n < 1) {
        set_error("%s: need 1 <= B <= 65535 samples of n >= 1 elements (B %d, n %lld)", what, B, n);
        return -1;
    }
    if (n > kQuantileMaxN) {
        set_error("quantile() input tensor is too large");
        return -1;
    }
    if (x == nullptr || out == nullptr) {
        set_error("%s: x and the quantile output are required", what);
        return -1;
    }
    const long long need = t2v_abs_quantile_workspace(B);
    if (ws == nullptr || ws_bytes < need) {
        set_error("%s: %d samples need a workspace of %lld bytes, got %lld", what, B, need, ws ? ws_bytes : 0LL);
        return -1;
    }
    return 0;
}
int t2v_abs_quantile(const float* x, int B, long long n, float q, float* out, void* workspace, long long workspace_bytes,
                     void* stream) {
    if (check_quantile_args("abs_quantile", x, B, n, out, workspace, workspace_bytes) != 0) return -1;
    if (!(q >= 0.f && q <= 1.f)) {
        set_error("abs_quantile: q must lie in [0, 1], got %g", static_cast<double>(q));
        return -1;
    }
    clear_pending_error("abs_quantile");
    return abs_quantile(x, B, n, q, out, workspace, reinterpret_cast<cudaStream_t>(stream));
}
int t2v_ddim_step_threshold(const float* x, const void* eps_c, const void* eps_u, int eps_is_f32, float* x_out, long long n,
                            long long chan_stride, int C, int guided_channels, float g, float a0, float a1, float a2, float a3,
                            float a4, const float* noise, int cfg_fp16, int B, float percentile, float* s_out, void* workspace,
                            long long workspace_bytes, void* stream) {
    if (x == nullptr || eps_c == nullptr || x_out == nullptr || x_out == x || n < 1 || chan_stride < 1 || C < 1) {
        set_error("ddim_step_threshold: x, eps_c and a distinct x_out are required, with n, chan_stride and C >= 1");
        return -1;
    }
    if (B < 1 || n % B != 0) {
        set_error("ddim_step_threshold: %lld elements do not split into %d samples", n, B);
        return -1;
    }
    if (!(percentile >= 0.f && percentile <= 1.f)) {
        set_error("ddim_step_threshold: percentile must be 0 (clamp) or lie in (0, 1], got %g", static_cast<double>(percentile));
        return -1;
    }
    if (percentile > 0.f && check_quantile_args("ddim_step_threshold", x, B, n / B, s_out, workspace, workspace_bytes) != 0)
        return -1;
    DdimStepParams p;
    p.x = x; p.eps_c = eps_c; p.eps_u = eps_u; p.eps_is_f32 = eps_is_f32;
    p.x_out = x_out; p.n = n; p.chan_stride = chan_stride; p.C = C; p.guided_channels = guided_channels; p.g = g;
    p.mode = 0; p.a0 = a0; p.a1 = a1; p.a2 = a2; p.a3 = a3; p.a4 = a4; p.noise = noise; p.cfg_fp16 = cfg_fp16;
    clear_pending_error("ddim_step_threshold");
    return ddim_threshold_step(p, B, percentile, s_out, workspace, reinterpret_cast<cudaStream_t>(stream));
}
int t2v_cfg_x0(const float* x, const void* eps_c, const void* eps_u, int eps_is_f32, float* x0, long long n, float g, float alpha,
               float sigma, int cfg_fp16, void* stream) {
    return cfg_x0(x, eps_c, eps_u, eps_is_f32, x0, n, g, alpha, sigma,
                  cfg_fp16, reinterpret_cast<cudaStream_t>(stream));
}
int t2v_lincomb(float* out, const float* const* src, const float* coef, int n_src, long long n, void* stream) {
    return lincomb(out, src, coef, n_src, n, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
