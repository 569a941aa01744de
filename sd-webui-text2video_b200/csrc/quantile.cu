// Exact per-sample quantile of |x| with torch.quantile's linear interpolation, by radix select on the fp32 bit patterns:
// with the sign cleared, non-negative floats (and the NaNs above +inf) order like their bits as uint32.  Three passes over the
// data select the lo-th and hi-th order statistics digit by digit (bits 30-20, 19-9, 8-0).  Each pass histograms the digit of
// every key whose higher bits match the prefix chosen so far; the last CTA of a sample to finish its pass (counted with an
// atomic ticket after a fence, so no grid barrier and no co-residency is needed) picks the bucket holding each target rank and
// clears the histogram for the next pass.  Counts are integers, so the result is deterministic.  No host synchronisation,
// so the whole select can be captured in a CUDA graph.
#include "common.cuh"
#include "kernels.cuh"

#include <math_constants.h>

namespace t2v {

namespace {

constexpr int kQThreads = 512;
constexpr int kQBins = 2048;
constexpr int kQPasses = 3;
__constant__ int kQShift[kQPasses] = {20, 9, 0};
__constant__ int kQBitsOf[kQPasses] = {11, 11, 9};

struct QuantileState {        // per sample, at the head of its workspace slice
    unsigned prefix[2];       // key bits above the current digit of the lo-th / hi-th order statistic
    unsigned rank[2];         // that statistic's rank among the keys sharing its prefix
    unsigned nan;             // the sample holds a NaN
    unsigned done;            // CTAs of the current pass that have added their histogram
    float w;                  // lerp weight rank - lo
    unsigned pad;
};
constexpr size_t kQStateBytes = 64;
constexpr size_t kQSampleBytes = kQStateBytes + 2 * kQBins * sizeof(unsigned);

__device__ __forceinline__ unsigned abs_key(float v) { return __float_as_uint(v) & 0x7fffffffu; }

// Exclusive prefix of v over the CTA (kQThreads threads); *total receives the sum.
__device__ unsigned block_exclusive_scan(unsigned v, unsigned* warp_sums, unsigned* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    if (lane == 31) warp_sums[warp] = inc;
    __syncthreads();
    if (warp == 0) {
        unsigned s = lane < kQThreads / 32 ? warp_sums[lane] : 0u;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned t = __shfl_up_sync(0xffffffffu, s, o);
            if (lane >= o) s += t;
        }
        if (lane < kQThreads / 32) warp_sums[lane] = s;
    }
    __syncthreads();
    const unsigned before = (warp > 0 ? warp_sums[warp - 1] : 0u) + inc - v;
    *total = warp_sums[kQThreads / 32 - 1];
    __syncthreads();
    return before;
}

// The bucket of hist holding rank r: the last CTA's step of the select.  Writes (bucket, r - keys in lower buckets) to out.
__device__ void select_bucket(const unsigned* hist, unsigned r, unsigned* warp_sums, unsigned* out) {
    constexpr int per = kQBins / kQThreads;
    const int b0 = threadIdx.x * per;
    unsigned sum = 0;
#pragma unroll
    for (int j = 0; j < per; ++j) sum += hist[b0 + j];
    unsigned total;
    unsigned cum = block_exclusive_scan(sum, warp_sums, &total);
    if (r >= cum && r < cum + sum) {
        for (int j = 0; j < per; ++j) {
            const unsigned h = hist[b0 + j];
            if (r < cum + h) {
                out[0] = static_cast<unsigned>(b0 + j);
                out[1] = r - cum;
                break;
            }
            cum += h;
        }
    }
    __syncthreads();
}

__device__ __forceinline__ float torch_lerp(float a, float b, float w) {
    return w < 0.5f ? __fadd_rn(a, __fmul_rn(w, __fsub_rn(b, a))) : __fsub_rn(b, __fmul_rn(__fsub_rn(b, a), __fsub_rn(1.f, w)));
}

// grid (CTAs per sample, B); sample b is x[b * n, (b + 1) * n), its workspace slice ws + b * kQSampleBytes.
template <bool VEC>
__global__ void __launch_bounds__(kQThreads) abs_quantile_pass_kernel(const float* __restrict__ x, long long n, float q, int pass,
                                                                     unsigned char* ws, float* out) {
    __shared__ unsigned s_hist[2][kQBins];
    __shared__ unsigned s_warp[kQThreads / 32];
    __shared__ unsigned s_sel[2][2];
    __shared__ unsigned s_state[2];
    __shared__ bool s_last;
    const int b = blockIdx.y;
    QuantileState* st = reinterpret_cast<QuantileState*>(ws + b * kQSampleBytes);
    unsigned* g_hist = reinterpret_cast<unsigned*>(ws + b * kQSampleBytes + kQStateBytes);
    const float* xs = x + b * n;
    const int shift = kQShift[pass], bits = kQBitsOf[pass];
    const unsigned digit_mask = (1u << bits) - 1u;
    unsigned p0 = 0, p1 = 0;
    if (pass > 0) {
        p0 = st->prefix[0];
        p1 = st->prefix[1];
    }
    const bool same = p0 == p1;          // one histogram serves both targets
    for (int i = threadIdx.x; i < 2 * kQBins; i += kQThreads) (&s_hist[0][0])[i] = 0u;
    __syncthreads();

    bool nan = false;
    auto add = [&](float v) {
        const unsigned k = abs_key(v);
        if (pass == 0) {
            nan |= k > 0x7f800000u;
            atomicAdd(&s_hist[0][k >> shift], 1u);
        } else {
            const unsigned hi = k >> (shift + bits), d = (k >> shift) & digit_mask;
            if (hi == p0) atomicAdd(&s_hist[0][d], 1u);
            if (!same && hi == p1) atomicAdd(&s_hist[1][d], 1u);
        }
    };
    const long long stride = static_cast<long long>(gridDim.x) * kQThreads;
    if (VEC) {
        const float4* x4 = reinterpret_cast<const float4*>(xs);
        const long long n4 = n >> 2;
        for (long long i = blockIdx.x * static_cast<long long>(kQThreads) + threadIdx.x; i < n4; i += stride) {
            const float4 v = __ldg(x4 + i);
            add(v.x);
            add(v.y);
            add(v.z);
            add(v.w);
        }
    } else {
        for (long long i = blockIdx.x * static_cast<long long>(kQThreads) + threadIdx.x; i < n; i += stride) add(__ldg(xs + i));
    }
    if (pass == 0 && __any_sync(0xffffffffu, nan) && (threadIdx.x & 31) == 0) atomicOr(&st->nan, 1u);
    __syncthreads();
    const int used = same ? 1 : 2;
    for (int i = threadIdx.x; i < used * kQBins; i += kQThreads) {
        const unsigned c = (&s_hist[0][0])[i];
        if (c != 0u) atomicAdd(g_hist + i, c);
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(&st->done, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!s_last) return;

    // last CTA of this sample's pass: every other CTA's histogram is in g_hist
    __threadfence();
    for (int i = threadIdx.x; i < used * kQBins; i += kQThreads) {
        (&s_hist[0][0])[i] = __ldcg(g_hist + i);
        g_hist[i] = 0u;
    }
    if (threadIdx.x == 0) {
        if (pass == 0) {
            // torch.quantile: rank = q * (n - 1) in fp32, lo = floor, hi = ceil, weight rank - lo
            const float rank = __fmul_rn(q, static_cast<float>(n - 1));
            const unsigned lo = static_cast<unsigned>(floorf(rank)), hi = static_cast<unsigned>(ceilf(rank));
            s_state[0] = lo;
            s_state[1] = hi;
            st->w = __fsub_rn(rank, static_cast<float>(lo));
        } else {
            s_state[0] = st->rank[0];
            s_state[1] = st->rank[1];
        }
        st->done = 0u;
    }
    __syncthreads();
    for (int t = 0; t < 2; ++t) select_bucket(s_hist[same ? 0 : t], s_state[t], s_warp, s_sel[t]);
    if (threadIdx.x == 0) {
        const unsigned k0 = (p0 << bits) | s_sel[0][0], k1 = (p1 << bits) | s_sel[1][0];
        st->prefix[0] = k0;
        st->prefix[1] = k1;
        st->rank[0] = s_sel[0][1];
        st->rank[1] = s_sel[1][1];
        if (pass == kQPasses - 1) {
            // a sample with a NaN: torch.quantile returns NaN
            out[b] = __ldcg(&st->nan) ? CUDART_NAN_F : torch_lerp(__uint_as_float(k0), __uint_as_float(k1), st->w);
        }
    }
}

}  // namespace

size_t abs_quantile_workspace(int B) { return static_cast<size_t>(B > 0 ? B : 0) * kQSampleBytes; }

int abs_quantile(const float* x, int B, long long n, float q, float* out, void* ws, cudaStream_t stream) {
    unsigned char* w = static_cast<unsigned char*>(ws);
    if (cudaMemsetAsync(w, 0, abs_quantile_workspace(B), stream) != cudaSuccess) return launch_status("abs_quantile memset");
    // one CTA per 16 elements per thread, at most two CTAs per SM (their shared memory and registers allow two) over the batch
    const long long per_sample_cap = (2LL * num_sms() + B - 1) / B;
    long long ctas = (n + 16LL * kQThreads - 1) / (16LL * kQThreads);
    if (ctas > per_sample_cap) ctas = per_sample_cap;
    if (ctas < 1) ctas = 1;
    const dim3 grid(static_cast<unsigned>(ctas), static_cast<unsigned>(B));
    const bool vec = (reinterpret_cast<uintptr_t>(x) & 15) == 0 && n % 4 == 0;
    for (int pass = 0; pass < kQPasses; ++pass) {
        if (vec)
            abs_quantile_pass_kernel<true><<<grid, kQThreads, 0, stream>>>(x, n, q, pass, w, out);
        else
            abs_quantile_pass_kernel<false><<<grid, kQThreads, 0, stream>>>(x, n, q, pass, w, out);
        const int rc = launch_status("abs_quantile launch");
        if (rc != 0) return rc;
    }
    return 0;
}

}  // namespace t2v
