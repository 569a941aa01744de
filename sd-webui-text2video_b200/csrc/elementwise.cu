// HBM-bound glue kernels: layout ingest/egress, nearest-2x upsample, stride-2 gather, concat, time embedding,
// tiny-M linears, row softmax, transposes, uint8 frame conversion, weight packing, sampler updates.
// All are simple grid-stride kernels with 16-byte vector accesses where the layout allows.
#include "common.cuh"
#include "kernels.cuh"

#include <math_constants.h>

namespace t2v {

namespace {

inline int grid_for(long long n, int threads, int cap = 132 * 16) {
    long long b = (n + threads - 1) / threads;
    if (b > cap) b = cap;
    if (b < 1) b = 1;
    return static_cast<int>(b);
}
#define GRID_STRIDE(i, n) \
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < (n); \
         i += static_cast<long long>(gridDim.x) * blockDim.x)

// frames [frame0, frame0 + nframes) of the (b f) order of x [B, C, F, h, w] -> tok rows [nframes * h * w][ld]
__global__ void ingest_kernel(const void* x, int x_is_f32, __half* tok, long long ld, int cpad, int C, int F, int h, int w,
                              long long frame0, long long nframes, float scale) {
    const long long P = static_cast<long long>(h) * w;
    const long long rows = nframes * P;
    GRID_STRIDE(i, rows * cpad) {
        const long long r = i / cpad;
        const int c = static_cast<int>(i - r * cpad);
        float v = 0.f;
        if (c < C) {
            const long long p = r % P;
            const long long bf = frame0 + r / P;
            const int f = static_cast<int>(bf % F);
            const int b = static_cast<int>(bf / F);
            const long long src = ((static_cast<long long>(b) * C + c) * F + f) * P + p;
            v = x_is_f32 ? reinterpret_cast<const float*>(x)[src] : __half2float(reinterpret_cast<const __half*>(x)[src]);
            v *= scale;
        }
        tok[r * ld + c] = __float2half_rn(v);
    }
}

__global__ void egress_kernel(const __half* tok, long long ld, void* out, int out_is_f32, int B, int C, int F, int h,
                              int w) {
    const long long P = static_cast<long long>(h) * w;
    const long long n = static_cast<long long>(B) * C * F * P;
    GRID_STRIDE(i, n) {
        const long long p = i % P;
        long long t = i / P;
        const int f = static_cast<int>(t % F);
        t /= F;
        const int c = static_cast<int>(t % C);
        const int b = static_cast<int>(t / C);
        const __half v = tok[((static_cast<long long>(b) * F + f) * P + p) * ld + c];
        if (out_is_f32) reinterpret_cast<float*>(out)[i] = __half2float(v);
        else reinterpret_cast<__half*>(out)[i] = v;
    }
}

__global__ void upsample2x_kernel(const uint4* x, uint4* y, long long nframes, int h, int w, int C8) {
    const int H = 2 * h, W = 2 * w;
    const long long n = nframes * H * W * C8;
    GRID_STRIDE(i, n) {
        const int c = static_cast<int>(i % C8);
        long long t = i / C8;
        const int X = static_cast<int>(t % W);
        t /= W;
        const int Y = static_cast<int>(t % H);
        const long long f = t / H;
        y[i] = __ldg(x + ((f * h + (Y >> 1)) * w + (X >> 1)) * C8 + c);
    }
}

__global__ void im2col_s2_kernel(const uint4* x, uint4* col, long long nframes, int h, int w, int C8, int pad_lo) {
    // pad_lo = 1: symmetric padding 1 (Conv2d stride 2 padding 1); pad_lo = 0: the ldm Downsample's pad (0,1,0,1) + padding 0
    const int ho = pad_lo ? (h + 1) / 2 : h / 2, wo = pad_lo ? (w + 1) / 2 : w / 2;
    const long long n = nframes * ho * wo * 9 * C8;
    GRID_STRIDE(i, n) {
        const int c = static_cast<int>(i % C8);
        long long t = i / C8;
        const int tap = static_cast<int>(t % 9);
        t /= 9;
        const int xo = static_cast<int>(t % wo);
        t /= wo;
        const int yo = static_cast<int>(t % ho);
        const long long f = t / ho;
        const int yi = 2 * yo + tap / 3 - pad_lo;
        const int xi = 2 * xo + tap % 3 - pad_lo;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (yi >= 0 && yi < h && xi >= 0 && xi < w) v = __ldg(x + ((f * h + yi) * w + xi) * C8 + c);
        col[i] = v;
    }
}

__global__ void concat_kernel(const __half* a, long long lda, int Ca8, const __half* b, long long ldb, int Cb8,
                              __half* out, long long ldo, long long rows) {
    const int T8 = Ca8 + Cb8;
    GRID_STRIDE(i, rows * T8) {
        const long long r = i / T8;
        const int c = static_cast<int>(i - r * T8);
        uint4 v;
        if (c < Ca8) v = __ldg(reinterpret_cast<const uint4*>(a + r * lda) + c);
        else v = __ldg(reinterpret_cast<const uint4*>(b + r * ldb) + (c - Ca8));
        reinterpret_cast<uint4*>(out + r * ldo)[c] = v;
    }
}

__global__ void time_sinusoid_kernel(const float* t, __half* out, int B, int dim) {
    const int half_dim = dim / 2;
    GRID_STRIDE(i, static_cast<long long>(B) * dim) {
        const int b = static_cast<int>(i / dim);
        const int j = static_cast<int>(i % dim);
        float v = 0.f;
        if (j < 2 * half_dim) {
            const int k = j < half_dim ? j : j - half_dim;
            // torch.pow(10000, -k/half) in fp32, then outer product with t (t2v_model.py:509-511)
            const float freq = powf(10000.0f, -(static_cast<float>(k) / static_cast<float>(half_dim)));
            const float s = t[b] * freq;
            v = j < half_dim ? cosf(s) : sinf(s);
        }
        out[i] = __float2half_rn(v);
    }
}

// one warp per output feature n; loops over the (few) samples
__global__ void __launch_bounds__(256) small_linear_kernel(const __half* x, long long ldx, const __half* W,
                                                           const __half* bias, const __half* addend, __half* y,
                                                           long long ldy, int B, int N, int K, int silu_in) {
    const int lane = threadIdx.x & 31;
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (n >= N) return;
    const __half* wr = W + static_cast<long long>(n) * K;
    for (int b = 0; b < B; ++b) {
        float acc = 0.f;
        for (int k = lane * 8; k < K; k += 256) {
            const uint4 wv = __ldg(reinterpret_cast<const uint4*>(wr + k));
            const uint4 xv = __ldg(reinterpret_cast<const uint4*>(x + b * ldx + k));
            const __half* wh = reinterpret_cast<const __half*>(&wv);
            const __half* xh = reinterpret_cast<const __half*>(&xv);
#pragma unroll
            for (int e = 0; e < 8; ++e) {
                float xe = __half2float(xh[e]);
                if (silu_in) xe = __half2float(__float2half_rn(xe / (1.0f + __expf(-xe))));   // SiLU output is fp16 in the reference
                acc += xe * __half2float(wh[e]);
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
        if (lane == 0) {
            if (bias) acc += __half2float(bias[n]);
            float r = __half2float(__float2half_rn(acc));     // the Linear's own fp16 output
            if (addend) r += __half2float(addend[n]);
            y[b * ldy + n] = __float2half_rn(r);
        }
    }
}

__global__ void __launch_bounds__(256) softmax_rows_kernel(const __half* x, __half* y, long long rows, int cols,
                                                           float scale) {
    // one warp per row, fp32 math; the scaled logits are rounded to fp16 first (reference: w_ * c^-0.5 in fp16)
    const int lane = threadIdx.x & 31;
    const long long row = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const __half* xr = x + row * cols;
    float m = -CUDART_INF_F;
    for (int c = lane; c < cols; c += 32) m = fmaxf(m, __half2float(__float2half_rn(__half2float(xr[c]) * scale)));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int c = lane; c < cols; c += 32) s += __expf(__half2float(__float2half_rn(__half2float(xr[c]) * scale)) - m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float inv = 1.0f / s;
    __half* yr = y + row * cols;
    for (int c = lane; c < cols; c += 32)
        yr[c] = __float2half_rn(__expf(__half2float(__float2half_rn(__half2float(xr[c]) * scale)) - m) * inv);
}

__global__ void transpose_kernel(const __half* x, __half* y, int R, int C) {
    __shared__ __half tile[32][34];
    const long long base = static_cast<long long>(blockIdx.z) * R * C;
    const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
    for (int j = threadIdx.y; j < 32; j += 8) {
        const int r = r0 + j, c = c0 + threadIdx.x;
        if (r < R && c < C) tile[j][threadIdx.x] = x[base + static_cast<long long>(r) * C + c];
    }
    __syncthreads();
    for (int j = threadIdx.y; j < 32; j += 8) {
        const int c = c0 + j, r = r0 + threadIdx.x;
        if (r < R && c < C) y[base + static_cast<long long>(c) * R + r] = tile[threadIdx.x][j];
    }
}

__global__ void frames_to_u8_kernel(const __half* tok, long long ld, uint8_t* out, long long pixels) {
    GRID_STRIDE(i, pixels * 3) {
        const long long p = i / 3;
        const int c = static_cast<int>(i - p * 3);
        // t2v_pipeline.py:447-460: fp32 x*0.5+0.5, clamp [0,1], *255, numpy astype(uint8) truncates
        float v = __half2float(tok[p * ld + c]);
        v = __fadd_rn(__fmul_rn(v, 0.5f), 0.5f);
        v = fminf(fmaxf(v, 0.f), 1.f);
        out[i] = static_cast<uint8_t>(__fmul_rn(v, 255.0f));
    }
}

// nn.PixelUnshuffle(8) of NCHW frames straight into tokens: row (n, y, x), column c*64 + i*8 + j = x[n, c, 8y+i, 8x+j].
// One thread per 8 consecutive columns (a fixed (c, i), j = 0..7): eight contiguous source pixels, one 16-byte store.
__global__ void pixel_unshuffle_kernel(const void* x, int x_is_f32, __half* tok, int N, int Cc, int H, int W) {
    const int h8 = H / 8, w8 = W / 8;
    const int groups = Cc * 8;                  // 8-column groups per row
    const long long n = static_cast<long long>(N) * h8 * w8 * groups;
    GRID_STRIDE(i, n) {
        const int g = static_cast<int>(i % groups);
        long long t = i / groups;
        const int xo = static_cast<int>(t % w8);
        t /= w8;
        const int yo = static_cast<int>(t % h8);
        const long long f = t / h8;
        const int c = g >> 3, ky = g & 7;
        const long long src = ((f * Cc + c) * H + (8 * yo + ky)) * static_cast<long long>(W) + 8 * xo;
        uint4 o;
        __half* oh = reinterpret_cast<__half*>(&o);
#pragma unroll
        for (int j = 0; j < 8; ++j)
            oh[j] = x_is_f32 ? __float2half_rn(reinterpret_cast<const float*>(x)[src + j]) : reinterpret_cast<const __half*>(x)[src + j];
        reinterpret_cast<uint4*>(tok)[i] = o;
    }
}

// y = max(x, 0) in place on a token matrix (n8 16-byte vectors); a NaN stays NaN, as nn.ReLU (__hmax2 would give 0)
__global__ void relu_kernel(uint4* x, long long n8) {
    const __half2 z = __float2half2_rn(0.f);
    GRID_STRIDE(i, n8) {
        uint4 v = x[i];
        __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
        for (int k = 0; k < 4; ++k) h[k] = __hmax2_nan(h[k], z);
        x[i] = v;
    }
}

// 2x2 average pooling, stride 2, floor sizes (nn.AvgPool2d(2, 2)): x [n, h, w, C] -> y [n, h/2, w/2, C]; fp32 sum of the four
// taps, times 0.25, one fp16 rounding
__global__ void avgpool2x2_kernel(const uint4* x, uint4* y, long long nframes, int h, int w, int C8) {
    const int ho = h / 2, wo = w / 2;
    GRID_STRIDE(i, nframes * ho * wo * C8) {
        const int c = static_cast<int>(i % C8);
        long long t = i / C8;
        const int xo = static_cast<int>(t % wo);
        t /= wo;
        const int yo = static_cast<int>(t % ho);
        const long long f = t / ho;
        float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
        for (int tap = 0; tap < 4; ++tap) {
            const uint4 v = __ldg(x + ((f * h + 2 * yo + (tap >> 1)) * w + 2 * xo + (tap & 1)) * C8 + c);
            const __half2* hv = reinterpret_cast<const __half2*>(&v);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float2 a = __half22float2(hv[k]);
                acc[2 * k] += a.x;
                acc[2 * k + 1] += a.y;
            }
        }
        uint4 o;
        __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int k = 0; k < 4; ++k) oh[k] = __floats2half2_rn(acc[2 * k] * 0.25f, acc[2 * k + 1] * 0.25f);
        y[i] = o;
    }
}

// x[r, :] += f[(r / rows_per_sample % f_samples) * rows_per_sample + r % rows_per_sample, :]  in place; fp32 add, one rounding
__global__ void feature_add_kernel(__half* x, long long ldx, const __half* f, int C8, long long rows, long long rows_per_sample,
                                   int f_samples) {
    GRID_STRIDE(i, rows * C8) {
        const long long r = i / C8;
        const int c = static_cast<int>(i - r * C8);
        const long long s = r / rows_per_sample;
        const long long fr = (s % f_samples) * rows_per_sample + (r - s * rows_per_sample);
        uint4* xp = reinterpret_cast<uint4*>(x + r * ldx) + c;
        uint4 a = *xp;
        const uint4 b = __ldg(reinterpret_cast<const uint4*>(f + fr * (static_cast<long long>(C8) * 8)) + c);
        __half2* ah = reinterpret_cast<__half2*>(&a);
        const __half2* bh = reinterpret_cast<const __half2*>(&b);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 u = __half22float2(ah[k]), v = __half22float2(bh[k]);
            ah[k] = __floats2half2_rn(u.x + v.x, u.y + v.y);
        }
        *xp = a;
    }
}

__global__ void frames_to_f32_kernel(const __half* tok, long long ld, float* out, int n, int H, int W) {
    const long long P = static_cast<long long>(H) * W;
    GRID_STRIDE(i, static_cast<long long>(n) * 3 * P) {
        const long long p = i % P;
        const long long t = i / P;
        const int c = static_cast<int>(t % 3);
        const long long f = t / 3;
        out[i] = __half2float(tok[(f * P + p) * ld + c]);
    }
}

__global__ void pack_conv_kernel(const void* src, int src_is_f32, __half* dst, int Cout, int Cin, int taps, int n_alloc,
                                 int k_alloc) {
    const long long n = static_cast<long long>(taps) * n_alloc * k_alloc;
    GRID_STRIDE(i, n) {
        const int k = static_cast<int>(i % k_alloc);
        long long t = i / k_alloc;
        const int o = static_cast<int>(t % n_alloc);
        const int tap = static_cast<int>(t / n_alloc);
        float v = 0.f;
        if (o < Cout && k < Cin) {
            const long long s = (static_cast<long long>(o) * Cin + k) * taps + tap;
            v = src_is_f32 ? reinterpret_cast<const float*>(src)[s] : __half2float(reinterpret_cast<const __half*>(src)[s]);
        }
        dst[i] = __float2half_rn(v);
    }
}

__global__ void pack_geglu_kernel(const void* w, const void* b, int src_is_f32, __half* wdst, __half* bdst, int H, int K,
                                  int bn) {
    // packed row p: tile = p / bn, j = p % bn ; j < bn/2 -> value channel tile*bn/2 + j ; else gate channel H + tile*bn/2 + (j - bn/2)
    const long long n = static_cast<long long>(2) * H * K;
    const int hb = bn / 2;
    GRID_STRIDE(i, n) {
        const int k = static_cast<int>(i % K);
        const int p = static_cast<int>(i / K);
        const int tile = p / bn, j = p % bn;
        const int srow = j < hb ? tile * hb + j : H + tile * hb + (j - hb);
        const long long s = static_cast<long long>(srow) * K + k;
        const float v = src_is_f32 ? reinterpret_cast<const float*>(w)[s] : __half2float(reinterpret_cast<const __half*>(w)[s]);
        wdst[i] = __float2half_rn(v);
        if (k == 0 && b != nullptr)
            bdst[p] = __float2half_rn(src_is_f32 ? reinterpret_cast<const float*>(b)[srow]
                                                 : __half2float(reinterpret_cast<const __half*>(b)[srow]));
    }
}

__global__ void splitk_reduce_kernel(const float* part, int splits, long long split_stride, long long rows, int N8,
                                     const __half* bias, int bias_rows, long long bias_stride, const __half* residual,
                                     long long ldr, __half* out, long long ldo) {
    GRID_STRIDE(i, rows * N8) {
        const long long r = i / N8;
        const int c = static_cast<int>(i - r * N8) * 8;
        float acc[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = 0.f;
        for (int s = 0; s < splits; ++s) {                   // fixed order: deterministic
            const float4* p = reinterpret_cast<const float4*>(part + s * split_stride + r * (static_cast<long long>(N8) * 8) + c);
            const float4 a = __ldg(p), b = __ldg(p + 1);
            acc[0] += a.x; acc[1] += a.y; acc[2] += a.z; acc[3] += a.w;
            acc[4] += b.x; acc[5] += b.y; acc[6] += b.z; acc[7] += b.w;
        }
        if (bias != nullptr) {
            const __half* bp = bias + (bias_rows > 0 ? (r / bias_rows) * bias_stride : 0) + c;
            const uint4 bv = __ldg(reinterpret_cast<const uint4*>(bp));
            const __half* bh = reinterpret_cast<const __half*>(&bv);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] += __half2float(bh[e]);
        }
        if (residual != nullptr) {
            const uint4 rv = __ldg(reinterpret_cast<const uint4*>(residual + r * ldr + c));
            const __half* rh = reinterpret_cast<const __half*>(&rv);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[e] += __half2float(rh[e]);
        }
        uint4 o;
        __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int e = 0; e < 4; ++e) oh[e] = __floats2half2_rn(acc[2 * e], acc[2 * e + 1]);
        *reinterpret_cast<uint4*>(out + r * ldo + c) = o;
    }
}

// one warp per output row n
__global__ void __launch_bounds__(256) fold_ln_kernel(const __half* w, const __half* bias, const __half* gamma, const __half* beta,
                                                      __half* wout, float* colsum, float* bias32, int N, int K) {
    const int lane = threadIdx.x & 31;
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (n >= N) return;
    float cs = 0.f, bs = 0.f;
    for (int k = lane; k < K; k += 32) {
        const float wv = __half2float(w[static_cast<long long>(n) * K + k]);
        const __half ws = __float2half_rn(wv * __half2float(gamma[k]));
        wout[static_cast<long long>(n) * K + k] = ws;
        cs += __half2float(ws);                 // column sum of EXACTLY what the tensor cores will multiply by
        bs += wv * __half2float(beta[k]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        cs += __shfl_xor_sync(0xffffffffu, cs, o);
        bs += __shfl_xor_sync(0xffffffffu, bs, o);
    }
    if (lane == 0) {
        colsum[n] = cs;
        bias32[n] = bs + (bias != nullptr ? __half2float(bias[n]) : 0.f);
    }
}

__global__ void convert_kernel(const void* src, int src_is_f32, __half* dst, long long n) {
    GRID_STRIDE(i, n) {
        dst[i] = src_is_f32 ? __float2half_rn(reinterpret_cast<const float*>(src)[i]) : reinterpret_cast<const __half*>(src)[i];
    }
}

__device__ __forceinline__ float cfg_combine(float c, float u, float g, int fp16) {
    if (fp16) {
        // u + g*(c - u) evaluated op by op in fp16, as torch does on fp16 tensors under autocast
        const float d = __half2float(__float2half_rn(c - u));
        const float s = __half2float(__float2half_rn(g * d));
        return __half2float(__float2half_rn(u + s));
    }
    return __fadd_rn(u, __fmul_rn(g, __fsub_rn(c, u)));
}

__device__ __forceinline__ float load_eps(const void* p, long long i, int is_f32) {
    return is_f32 ? reinterpret_cast<const float*>(p)[i] : __half2float(reinterpret_cast<const __half*>(p)[i]);
}

// VideoCrafter's uc_type formulas (lvdm/samplers/ddim.py:233-241) in fp32, op by op; kVariant 0 is cfg_combine itself.
// The host allows kVariant 1 and 2 only with fp16 == 0.
template <int kVariant>
__device__ __forceinline__ float cfg_variant(float c, float u, float g, int fp16) {
    if constexpr (kVariant == 1) return __fadd_rn(c, __fmul_rn(g, __fsub_rn(c, u)));     // 'cfg_original'
    else if constexpr (kVariant == 2) return __fadd_rn(c, __fmul_rn(g, __fsub_rn(u, c)));   // 'cfg_ours'
    else return cfg_combine(c, u, g, fp16);
}

// kX0: also store mode 1's x0 (the value the update uses) to x0_out; the host allows it only in mode 1.
// <false, 0> is the kernel t2v_ddim_step has always launched; x0_out is unused there.
template <bool kX0, int kVariant>
__global__ void ddim_step_kernel(DdimStepParams p, float* x0_out) {
    GRID_STRIDE(i, p.n) {
        const int ch = static_cast<int>((i / p.chan_stride) % p.C);
        const float c = load_eps(p.eps_c, i, p.eps_is_f32);
        float e = c;
        if (p.eps_u != nullptr && ch < p.guided_channels)
            e = cfg_variant<kVariant>(c, load_eps(p.eps_u, i, p.eps_is_f32), p.g, p.cfg_fp16);
        const float x = p.x[i];
        const float nz = (p.noise != nullptr && p.a4 != 0.f) ? __fmul_rn(p.a4, p.noise[i]) : 0.f;
        float xn;
        if (p.mode == 0) {
            const float ax = __fmul_rn(p.a0, x);
            const float x0 = __fsub_rn(ax, __fmul_rn(p.a1, e));
            const float eps = __fdiv_rn(__fsub_rn(ax, x0), p.a1);
            xn = __fadd_rn(__fadd_rn(__fmul_rn(p.a2, x0), __fmul_rn(p.a3, eps)), nz);
        } else {
            const float x0 = __fdiv_rn(__fsub_rn(x, __fmul_rn(p.a0, e)), p.a1);
            if constexpr (kX0) x0_out[i] = x0;
            xn = __fadd_rn(__fadd_rn(__fmul_rn(p.a2, x0), __fmul_rn(p.a3, e)), nz);
        }
        p.x_out[i] = xn;
    }
}

// torch.maximum / torch.minimum / torch.clamp: a NaN operand gives NaN
__device__ __forceinline__ float nan_max(float a, float b) { return isnan(a) ? a : (isnan(b) ? b : fmaxf(a, b)); }
__device__ __forceinline__ float nan_min(float a, float b) { return isnan(a) ? a : (isnan(b) ? b : fminf(a, b)); }

// DDIM_Gaussian's x0 (mode 0 of ddim_step_kernel) -> x_out, the input of the dynamic-thresholding quantile
__global__ void ddim_x0_kernel(DdimStepParams p) {
    GRID_STRIDE(i, p.n) {
        const int ch = static_cast<int>((i / p.chan_stride) % p.C);
        const float c = load_eps(p.eps_c, i, p.eps_is_f32);
        float e = c;
        if (p.eps_u != nullptr && ch < p.guided_channels) e = cfg_combine(c, load_eps(p.eps_u, i, p.eps_is_f32), p.g, p.cfg_fp16);
        p.x_out[i] = __fsub_rn(__fmul_rn(p.a0, p.x[i]), __fmul_rn(p.a1, e));
    }
}

// Mode 0 with x0 restricted before eps is recomputed from it (gaussian_sampler.py:110-120, :174-178, :199-202):
// s != null: x0 = min(s', max(-s', x0)) / s' with s' = max(s[sample], 1); s == null: x0 = clamp(x0, -1, 1).
__global__ void ddim_threshold_kernel(DdimStepParams p, const float* s, long long sample_n) {
    GRID_STRIDE(i, p.n) {
        const int ch = static_cast<int>((i / p.chan_stride) % p.C);
        const float c = load_eps(p.eps_c, i, p.eps_is_f32);
        float e = c;
        if (p.eps_u != nullptr && ch < p.guided_channels) e = cfg_combine(c, load_eps(p.eps_u, i, p.eps_is_f32), p.g, p.cfg_fp16);
        const float x = p.x[i];
        const float nz = (p.noise != nullptr && p.a4 != 0.f) ? __fmul_rn(p.a4, p.noise[i]) : 0.f;
        const float ax = __fmul_rn(p.a0, x);
        float x0 = __fsub_rn(ax, __fmul_rn(p.a1, e));
        if (s != nullptr) {
            const float si = nan_max(s[i / sample_n], 1.f);
            x0 = __fdiv_rn(nan_min(si, nan_max(-si, x0)), si);
        } else {
            x0 = nan_min(nan_max(x0, -1.f), 1.f);
        }
        const float eps = __fdiv_rn(__fsub_rn(ax, x0), p.a1);
        p.x_out[i] = __fadd_rn(__fadd_rn(__fmul_rn(p.a2, x0), __fmul_rn(p.a3, eps)), nz);
    }
}

struct LincombArgs {
    const float* src[8];
    float coef[8];
    int n_src;
};
__global__ void lincomb_kernel(float* out, LincombArgs a, long long n) {
    GRID_STRIDE(i, n) {
        float acc = 0.f;
        for (int s = 0; s < a.n_src; ++s) acc = fmaf(a.coef[s], a.src[s][i], acc);
        out[i] = acc;
    }
}

__global__ void cfg_x0_kernel(const float* x, const void* ec, const void* eu, int eps_f32, float* x0, long long n, float g,
                              float alpha, float sigma, int fp16) {
    GRID_STRIDE(i, n) {
        float e = load_eps(ec, i, eps_f32);
        if (eu != nullptr) e = cfg_combine(e, load_eps(eu, i, eps_f32), g, fp16);
        x0[i] = __fdiv_rn(__fsub_rn(x[i], __fmul_rn(sigma, e)), alpha);
    }
}

// img2vid inpainting latent (process_modelscope.py:209: masked = image_latents * (1 - mask) + latent_noise * mask, numpy
// float64 with a per-frame mask weight): out[b,c,f,p] = img[b,c,f or 0,p] * (1 - w[f]) + noise[b,c,f,p] * w[f]
__global__ void latent_blend_kernel(const float* __restrict__ img, int img_frames, const double* __restrict__ noise,
                                    const double* __restrict__ w, double* __restrict__ out, double* __restrict__ mask, long long n,
                                    int F, long long hw) {
    GRID_STRIDE(i, n) {
        const long long bc = i / (static_cast<long long>(F) * hw);
        const long long r = i - bc * F * hw;
        const int f = static_cast<int>(r / hw);
        const long long p = r - static_cast<long long>(f) * hw;
        const double m = w[f];
        const double a = static_cast<double>(img[(bc * img_frames + (img_frames == 1 ? 0 : f)) * hw + p]);
        out[i] = __dadd_rn(__dmul_rn(a, __dsub_rn(1.0, m)), __dmul_rn(noise[i], m));
        if (mask != nullptr) mask[i] = m;
    }
}

// VideoCrafter q_sample / masked DDIM blend (videocrafter/lvdm/models/ddpm3d.py:283-286, lvdm/samplers/ddim.py:188-195) in
// torch's fp32 op order, no contraction: known = a[b]*x0 + s[b]*noise; out = known*mask + (1 - mask)*img when blending.
// x0 / noise / mask are read through element strides (0 on a broadcast dimension); img and out are contiguous.
__global__ void q_sample_blend_kernel(QSampleBlendParams p) {
    const long long hw = static_cast<long long>(p.shape[3]) * p.shape[4];
    const long long n = static_cast<long long>(p.shape[0]) * p.shape[1] * p.shape[2] * hw;
    GRID_STRIDE(i, n) {
        const int x = static_cast<int>(i % p.shape[4]);
        long long r = i / p.shape[4];
        const int y = static_cast<int>(r % p.shape[3]);
        r /= p.shape[3];
        const int t = static_cast<int>(r % p.shape[2]);
        r /= p.shape[2];
        const int c = static_cast<int>(r % p.shape[1]);
        const int b = static_cast<int>(r / p.shape[1]);
        const int idx[5] = {b, c, t, y, x};
        long long ox = 0, on = 0, om = 0;
#pragma unroll
        for (int d = 0; d < 5; ++d) {
            ox += idx[d] * p.x0_stride[d];
            on += idx[d] * p.noise_stride[d];
            om += idx[d] * p.mask_stride[d];
        }
        const float known = __fadd_rn(__fmul_rn(p.a[b], p.x0[ox]), __fmul_rn(p.s[b], p.noise[on]));
        if (p.mask == nullptr) {
            p.out[i] = known;
        } else {
            const float m = p.mask[om];
            p.out[i] = __fadd_rn(__fmul_rn(known, m), __fmul_rn(__fsub_rn(1.0f, m), p.img[i]));
        }
    }
}

// LoRA hot-merge (stable_lora/stable_utils/lora_processor.py:50-96 under autocast): the low-rank product is formed with fp32
// accumulation and rounded to fp16 (torch's autocast matmul), scaled by alpha in fp16, added in fp16.
__global__ void lora_merge_kernel(__half* __restrict__ w, const __half* __restrict__ A, const __half* __restrict__ B, int out, int cols,
                                  int rank, float alpha, int temporal_mean) {
    const long long n = static_cast<long long>(out) * cols;
    const int a_cols = temporal_mean ? cols * 3 : cols;
    GRID_STRIDE(i, n) {
        const int o = static_cast<int>(i / cols);
        const int j = static_cast<int>(i - static_cast<long long>(o) * cols);
        float d;
        if (temporal_mean) {
            float sum = 0.f;
            for (int q = 0; q < 3; ++q) {
                float acc = 0.f;
                for (int r = 0; r < rank; ++r)
                    acc = fmaf(__half2float(B[static_cast<long long>(o) * rank + r]), __half2float(A[static_cast<long long>(r) * a_cols + j * 3 + q]), acc);
                sum += __half2float(__float2half_rn(acc));
            }
            d = __half2float(__float2half_rn(sum / 3.0f));            // torch.mean on fp16: fp32 accumulate, divide, round
        } else {
            float acc = 0.f;
            for (int r = 0; r < rank; ++r)
                acc = fmaf(__half2float(B[static_cast<long long>(o) * rank + r]), __half2float(A[static_cast<long long>(r) * a_cols + j]), acc);
            d = __half2float(__float2half_rn(acc));
        }
        const float scaled = __half2float(__float2half_rn(d * alpha));
        w[i] = __float2half_rn(__half2float(w[i]) + scaled);
    }
}

// VideoCrafter LoRA merge (videocrafter/lvdm/models/modules/lora.py:650-666, `weight.data += alpha * torch.mm(up, down)` on an
// fp16 weight): the product is accumulated in fp32 from fp32 (or exactly widened fp16) factors, scaled in fp32, added to the
// widened weight in fp32, and rounded to fp16 once.
__device__ __forceinline__ float widen(float v) { return v; }
__device__ __forceinline__ float widen(__half v) { return __half2float(v); }

template <class T>
__global__ void lora_apply_kernel(__half* __restrict__ w, const T* __restrict__ up, const T* __restrict__ down, int out, int cols,
                                  int rank, float alpha) {
    const long long n = static_cast<long long>(out) * cols;
    GRID_STRIDE(i, n) {
        const int o = static_cast<int>(i / cols);
        const int j = static_cast<int>(i - static_cast<long long>(o) * cols);
        float acc = 0.f;
        for (int r = 0; r < rank; ++r)
            acc = fmaf(widen(up[static_cast<long long>(o) * rank + r]), widen(down[static_cast<long long>(r) * cols + j]), acc);
        w[i] = __float2half_rn(__fadd_rn(__half2float(w[i]), __fmul_rn(alpha, acc)));
    }
}

inline int ok() { return launch_status("elementwise launch"); }

}  // namespace

int ingest_latent(const void* x, int x_is_f32, __half* tok, long long ld, int cpad, int B, int C, int F, int h, int w,
                  float scale, cudaStream_t stream) {
    return ingest_latent_frames(x, x_is_f32, tok, ld, cpad, C, F, h, w, 0, static_cast<long long>(B) * F, scale, stream);
}
int ingest_latent_frames(const void* x, int x_is_f32, __half* tok, long long ld, int cpad, int C, int F, int h, int w,
                         long long frame0, long long nframes, float scale, cudaStream_t stream) {
    const long long n = nframes * h * w * cpad;
    ingest_kernel<<<grid_for(n, 256), 256, 0, stream>>>(x, x_is_f32, tok, ld, cpad, C, F, h, w, frame0, nframes, scale);
    return ok();
}
int egress_latent(const __half* tok, long long ld, void* out, int out_is_f32, int B, int C, int F, int h, int w,
                  cudaStream_t stream) {
    const long long n = static_cast<long long>(B) * C * F * h * w;
    egress_kernel<<<grid_for(n, 256), 256, 0, stream>>>(tok, ld, out, out_is_f32, B, C, F, h, w);
    return ok();
}
int upsample2x(const __half* x, __half* y, int nframes, int h, int w, int C, cudaStream_t stream) {
    if (C % 8) return -1;
    const long long n = static_cast<long long>(nframes) * 4 * h * w * (C / 8);
    upsample2x_kernel<<<grid_for(n, 256), 256, 0, stream>>>(reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(y),
                                                            nframes, h, w, C / 8);
    return ok();
}
int im2col_s2(const __half* x, __half* col, int nframes, int h, int w, int C, cudaStream_t stream, int pad_lo) {
    if (C % 8) return -1;
    const long long n = static_cast<long long>(nframes) * ((pad_lo ? (h + 1) / 2 : h / 2)) * ((pad_lo ? (w + 1) / 2 : w / 2)) * 9 * (C / 8);
    im2col_s2_kernel<<<grid_for(n, 256), 256, 0, stream>>>(reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(col),
                                                           nframes, h, w, C / 8, pad_lo);
    return ok();
}
int pixel_unshuffle_ingest(const void* x, int x_is_f32, __half* tok, int N, int Cc, int H, int W, cudaStream_t stream) {
    if (H % 8 || W % 8) return -1;
    const long long n = static_cast<long long>(N) * (H / 8) * (W / 8) * Cc * 8;
    pixel_unshuffle_kernel<<<grid_for(n, 256), 256, 0, stream>>>(x, x_is_f32, tok, N, Cc, H, W);
    return ok();
}
int relu_inplace(__half* x, long long rows, int C, cudaStream_t stream) {
    if (C % 8) return -1;
    const long long n8 = rows * (C / 8);
    relu_kernel<<<grid_for(n8, 256), 256, 0, stream>>>(reinterpret_cast<uint4*>(x), n8);
    return ok();
}
int avgpool2x2(const __half* x, __half* y, int nframes, int h, int w, int C, cudaStream_t stream) {
    if (C % 8) return -1;
    const long long n = static_cast<long long>(nframes) * (h / 2) * (w / 2) * (C / 8);
    avgpool2x2_kernel<<<grid_for(n, 256), 256, 0, stream>>>(reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(y),
                                                            nframes, h, w, C / 8);
    return ok();
}
int feature_add(__half* x, long long ldx, const __half* f, int C, long long rows, long long rows_per_sample, int f_samples,
                cudaStream_t stream) {
    if (C % 8 || ldx % 8 || rows_per_sample < 1 || f_samples < 1) return -1;
    const long long n = rows * (C / 8);
    feature_add_kernel<<<grid_for(n, 256), 256, 0, stream>>>(x, ldx, f, C / 8, rows, rows_per_sample, f_samples);
    return ok();
}
int concat_cols(const __half* a, long long lda, int Ca, const __half* b, long long ldb, int Cb, __half* out,
                long long ldo, long long rows, cudaStream_t stream) {
    if ((Ca % 8) || (Cb % 8) || (lda % 8) || (ldb % 8) || (ldo % 8)) return -1;
    const long long n = rows * ((Ca + Cb) / 8);
    concat_kernel<<<grid_for(n, 256), 256, 0, stream>>>(a, lda, Ca / 8, b, ldb, Cb / 8, out, ldo, rows);
    return ok();
}
int time_sinusoid(const float* t, __half* out, int B, int dim, cudaStream_t stream) {
    time_sinusoid_kernel<<<grid_for(static_cast<long long>(B) * dim, 256), 256, 0, stream>>>(t, out, B, dim);
    return ok();
}
int small_linear(const __half* x, long long ldx, const __half* W, const __half* bias, const __half* addend, __half* y,
                 long long ldy, int B, int N, int K, int silu_in, cudaStream_t stream) {
    if ((K % 8) || (ldx % 8)) return -1;
    small_linear_kernel<<<(N + 7) / 8, 256, 0, stream>>>(x, ldx, W, bias, addend, y, ldy, B, N, K, silu_in);
    return ok();
}
int softmax_rows(const __half* x, __half* y, long long rows, int cols, float scale, cudaStream_t stream) {
    softmax_rows_kernel<<<static_cast<unsigned int>((rows + 7) / 8), 256, 0, stream>>>(x, y, rows, cols, scale);
    return ok();
}
int transpose_batched(const __half* x, __half* y, int nb, int R, int C, cudaStream_t stream) {
    dim3 grid((C + 31) / 32, (R + 31) / 32, nb);
    transpose_kernel<<<grid, dim3(32, 8), 0, stream>>>(x, y, R, C);
    return ok();
}
int frames_to_u8(const __half* tok, long long ld, uint8_t* out, long long pixels, cudaStream_t stream) {
    frames_to_u8_kernel<<<grid_for(pixels * 3, 256), 256, 0, stream>>>(tok, ld, out, pixels);
    return ok();
}
int frames_to_f32_nchw(const __half* tok, long long ld, float* out, int n, int H, int W, cudaStream_t stream) {
    frames_to_f32_kernel<<<grid_for(static_cast<long long>(n) * 3 * H * W, 256), 256, 0, stream>>>(tok, ld, out, n, H, W);
    return ok();
}
int pack_conv_weight(const void* src, int src_is_f32, __half* dst, int Cout, int Cin, int taps, int n_alloc, int k_alloc,
                     cudaStream_t stream) {
    const long long n = static_cast<long long>(taps) * n_alloc * k_alloc;
    pack_conv_kernel<<<grid_for(n, 256), 256, 0, stream>>>(src, src_is_f32, dst, Cout, Cin, taps, n_alloc, k_alloc);
    return ok();
}
int pack_geglu_weight(const void* w, const void* b, int src_is_f32, __half* wdst, __half* bdst, int H, int K, int bn,
                      cudaStream_t stream) {
    if ((2 * H) % bn) return -1;
    pack_geglu_kernel<<<grid_for(static_cast<long long>(2) * H * K, 256), 256, 0, stream>>>(w, b, src_is_f32, wdst, bdst, H, K, bn);
    return ok();
}
int splitk_reduce(const float* part, int splits, long long split_stride, long long rows, int N, const __half* bias,
                  int bias_rows, long long bias_stride, const __half* residual, long long ldr, __half* out, long long ldo,
                  cudaStream_t stream) {
    if ((N & 7) || (ldo & 7) || (residual && (ldr & 7)) || (bias && (bias_stride & 7))) return -1;
    splitk_reduce_kernel<<<grid_for(rows * (N / 8), 256), 256, 0, stream>>>(part, splits, split_stride, rows, N / 8, bias,
                                                                            bias_rows, bias_stride, residual, ldr, out, ldo);
    return ok();
}
int fold_ln_into_linear(const __half* w, const __half* bias, const __half* gamma, const __half* beta, __half* wout,
                        float* colsum, float* bias32, int N, int K, cudaStream_t stream) {
    fold_ln_kernel<<<(N + 7) / 8, 256, 0, stream>>>(w, bias, gamma, beta, wout, colsum, bias32, N, K);
    return ok();
}
int convert_to_f16(const void* src, int src_is_f32, __half* dst, long long n, cudaStream_t stream) {
    convert_kernel<<<grid_for(n, 256), 256, 0, stream>>>(src, src_is_f32, dst, n);
    return ok();
}
template <int kVariant>
static void launch_ddim_step(const DdimStepParams& p, float* x0_out, cudaStream_t stream) {
    if (x0_out != nullptr)
        ddim_step_kernel<true, kVariant><<<grid_for(p.n, 256), 256, 0, stream>>>(p, x0_out);
    else
        ddim_step_kernel<false, kVariant><<<grid_for(p.n, 256), 256, 0, stream>>>(p, nullptr);
}
int ddim_step(const DdimStepParams& p, int cfg_variant, float* x0_out, cudaStream_t stream) {
    switch (cfg_variant) {
        case 0: launch_ddim_step<0>(p, x0_out, stream); break;
        case 1: launch_ddim_step<1>(p, x0_out, stream); break;
        case 2: launch_ddim_step<2>(p, x0_out, stream); break;
        default: return -1;
    }
    return ok();
}
int ddim_threshold_step(const DdimStepParams& p, int B, float percentile, float* s, void* ws, cudaStream_t stream) {
    if (percentile > 0.f) {
        ddim_x0_kernel<<<grid_for(p.n, 256), 256, 0, stream>>>(p);
        int rc = ok();
        if (rc != 0) return rc;
        if ((rc = abs_quantile(p.x_out, B, p.n / B, percentile, s, ws, stream)) != 0) return rc;
    }
    ddim_threshold_kernel<<<grid_for(p.n, 256), 256, 0, stream>>>(p, percentile > 0.f ? s : nullptr, p.n / B);
    return ok();
}
int lincomb(float* out, const float* const* src, const float* coef, int n_src, long long n, cudaStream_t stream) {
    if (n_src < 1 || n_src > 8) return -1;
    LincombArgs a;
    for (int i = 0; i < n_src; ++i) {
        a.src[i] = src[i];
        a.coef[i] = coef[i];
    }
    a.n_src = n_src;
    lincomb_kernel<<<grid_for(n, 256), 256, 0, stream>>>(out, a, n);
    return ok();
}
int lora_merge_weight(__half* w, const __half* A, const __half* B, int out, int cols, int rank, float alpha, int temporal_mean,
                      cudaStream_t stream) {
    const long long n = static_cast<long long>(out) * cols;
    lora_merge_kernel<<<grid_for(n, 256), 256, 0, stream>>>(w, A, B, out, cols, rank, alpha, temporal_mean);
    return ok();
}
int lora_apply_weight(__half* w, const void* up, const void* down, int dtype, int out, int cols, int rank, float alpha,
                      cudaStream_t stream) {
    const long long n = static_cast<long long>(out) * cols;
    if (dtype == 1)
        lora_apply_kernel<float><<<grid_for(n, 256), 256, 0, stream>>>(w, static_cast<const float*>(up),
                                                                       static_cast<const float*>(down), out, cols, rank, alpha);
    else
        lora_apply_kernel<__half><<<grid_for(n, 256), 256, 0, stream>>>(w, static_cast<const __half*>(up),
                                                                        static_cast<const __half*>(down), out, cols, rank, alpha);
    return ok();
}

int latent_blend(const float* img, int img_frames, const double* noise, const double* w, double* out, double* mask, int BC, int F,
                 long long hw, cudaStream_t stream) {
    const long long n = static_cast<long long>(BC) * F * hw;
    latent_blend_kernel<<<grid_for(n, 256), 256, 0, stream>>>(img, img_frames, noise, w, out, mask, n, F, hw);
    return ok();
}

int q_sample_blend(const QSampleBlendParams& p, cudaStream_t stream) {
    const long long n = static_cast<long long>(p.shape[0]) * p.shape[1] * p.shape[2] * p.shape[3] * p.shape[4];
    q_sample_blend_kernel<<<grid_for(n, 256), 256, 0, stream>>>(p);
    return ok();
}

int cfg_x0(const float* x, const void* eps_c, const void* eps_u, int eps_is_f32, float* x0, long long n, float g,
           float alpha, float sigma, int cfg_fp16, cudaStream_t stream) {
    cfg_x0_kernel<<<grid_for(n, 256), 256, 0, stream>>>(x, eps_c, eps_u, eps_is_f32, x0, n, g, alpha, sigma, cfg_fp16);
    return ok();
}

}  // namespace t2v
