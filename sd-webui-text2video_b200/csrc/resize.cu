// Frame preparation of vid2vid / img2vid (process_modelscope.py:115-137, :172-190): PIL's Image.resize((W, H), LANCZOS) of
// uint8 RGB frames, then the reference's x / 255 * 2 - 1, bit for bit.
//
// Pillow's resampler (libImaging/Resample.c) is integer arithmetic over coefficient tables built in double on the host:
//   scale = in / out, filterscale = max(scale, 1), support = 3 * filterscale, ksize = 2 * ceil(support) + 1;
//   output pixel xx: center = (xx + 0.5) * scale, first = max((int)(center - support + 0.5), 0),
//   last = min((int)(center + support + 0.5), in), w_x = lanczos((x + first - center + 0.5) * (1 / filterscale)),
//   normalised by their sum and rounded half away from zero to int32 with 22 fractional bits.
// The horizontal pass runs first, over the rows the vertical pass reads, into a uint8 image; each pass accumulates
// 2^21 + sum(pixel * k) in int32 and clips acc >> 22 to [0, 255].  A pass whose size does not change is skipped; here the
// vertical one then runs the identity table (one tap of weight 2^22), which carries the normalisation.
#include "common.cuh"
#include "kernels.cuh"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <map>
#include <mutex>
#include <tuple>
#include <vector>

namespace t2v {
namespace {

constexpr int kPrecisionBits = 22;

double sinc(double x) {
    if (x == 0.0) return 1.0;
    x *= M_PI;
    return sin(x) / x;
}

double lanczos(double x) { return (-3.0 <= x && x < 3.0) ? sinc(x) * sinc(x / 3.0) : 0.0; }

struct Table {
    int ksize = 0;
    std::vector<int> bounds;     // [out][2]: first input pixel, taps used
    std::vector<int> coeffs;     // [out][ksize], zero past the taps used
};

Table build_table(int in_size, int out_size) {
    Table t;
    t.bounds.resize(2 * static_cast<size_t>(out_size));
    if (in_size == out_size) {   // the pass Pillow skips
        t.ksize = 1;
        t.coeffs.assign(out_size, 1 << kPrecisionBits);
        for (int i = 0; i < out_size; ++i) {
            t.bounds[2 * i] = i;
            t.bounds[2 * i + 1] = 1;
        }
        return t;
    }
    const double scale = static_cast<double>(in_size) / out_size;
    const double filterscale = scale < 1.0 ? 1.0 : scale;
    const double support = 3.0 * filterscale;
    const double ss = 1.0 / filterscale;
    t.ksize = static_cast<int>(ceil(support)) * 2 + 1;
    t.coeffs.assign(static_cast<size_t>(out_size) * t.ksize, 0);
    std::vector<double> w(t.ksize);
    for (int xx = 0; xx < out_size; ++xx) {
        const double center = (xx + 0.5) * scale;
        int xmin = static_cast<int>(center - support + 0.5);
        if (xmin < 0) xmin = 0;
        int xmax = static_cast<int>(center + support + 0.5);
        if (xmax > in_size) xmax = in_size;
        xmax -= xmin;
        double ww = 0.0;
        for (int x = 0; x < xmax; ++x) {
            w[x] = lanczos((x + xmin - center + 0.5) * ss);
            ww += w[x];
        }
        int* k = &t.coeffs[static_cast<size_t>(xx) * t.ksize];
        for (int x = 0; x < xmax; ++x) {
            const double v = (ww != 0.0 ? w[x] / ww : w[x]) * (1 << kPrecisionBits);
            k[x] = static_cast<int>(v < 0 ? -0.5 + v : 0.5 + v);
        }
        t.bounds[2 * xx] = xmin;
        t.bounds[2 * xx + 1] = xmax;
    }
    return t;
}

struct DeviceTable {
    int ksize;
    int first, last;             // input pixels [first, last) any output reads
    const int2* bounds;
    const int* coeffs;
};

// One device copy of each (device, in, out) table, made on first use and kept for the life of the process.
int device_table(int in_size, int out_size, DeviceTable* out) {
    static std::mutex mu;
    static std::map<std::tuple<int, int, int>, DeviceTable> cache;
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return launch_status("frames_resize: cudaGetDevice");
    std::lock_guard<std::mutex> lock(mu);
    const auto key = std::make_tuple(dev, in_size, out_size);
    const auto it = cache.find(key);
    if (it != cache.end()) {
        *out = it->second;
        return 0;
    }
    const Table t = build_table(in_size, out_size);
    const size_t bb = t.bounds.size() * sizeof(int), cb = t.coeffs.size() * sizeof(int);
    char* d = nullptr;
    if (cudaMalloc(&d, bb + cb) != cudaSuccess) return launch_status("frames_resize: coefficient table allocation");
    if (cudaMemcpy(d, t.bounds.data(), bb, cudaMemcpyHostToDevice) != cudaSuccess ||
        cudaMemcpy(d + bb, t.coeffs.data(), cb, cudaMemcpyHostToDevice) != cudaSuccess) {
        cudaFree(d);
        return launch_status("frames_resize: coefficient table upload");
    }
    DeviceTable dt;
    dt.ksize = t.ksize;
    dt.first = t.bounds[0];
    dt.last = t.bounds[2 * (out_size - 1)] + t.bounds[2 * (out_size - 1) + 1];
    dt.bounds = reinterpret_cast<const int2*>(d);
    dt.coeffs = reinterpret_cast<const int*>(d + bb);
    cache.emplace(key, dt);
    *out = dt;
    return 0;
}

__device__ __forceinline__ uint8_t clip8(int acc) { return static_cast<uint8_t>(min(max(acc >> kPrecisionBits, 0), 255)); }

__device__ __forceinline__ void store(float* p, float v) { *p = v; }
__device__ __forceinline__ void store(__half* p, float v) { *p = __float2half_rn(v); }

// Horizontal pass: src rows [row0, row0 + rows) of every frame [H0, W0, 3] -> tmp [rows, W, 3]; one thread per output pixel.
__global__ void __launch_bounds__(128) resize_h_kernel(const uint8_t* __restrict__ src, long long src_frame, int W0, int row0,
                                                       int rows, const int2* __restrict__ bounds, const int* __restrict__ coeffs,
                                                       int ksize, uint8_t* __restrict__ tmp, int W, int n) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= W) return;
    const int2 b = __ldg(&bounds[x]);
    const int* k = coeffs + static_cast<long long>(x) * ksize;
    for (int f = blockIdx.z; f < n; f += gridDim.z) {
        const uint8_t* s = src + f * src_frame + (static_cast<long long>(row0 + y) * W0 + b.x) * 3;
        int a0 = 1 << (kPrecisionBits - 1), a1 = a0, a2 = a0;
        for (int j = 0; j < b.y; ++j) {
            const int kj = __ldg(&k[j]);
            a0 += s[3 * j] * kj;
            a1 += s[3 * j + 1] * kj;
            a2 += s[3 * j + 2] * kj;
        }
        uint8_t* o = tmp + static_cast<long long>(f) * rows * W * 3 + (static_cast<long long>(y) * W + x) * 3;
        o[0] = clip8(a0);
        o[1] = clip8(a1);
        o[2] = clip8(a2);
    }
}

// Vertical pass + normalisation: src [*, W, 3] rows (bounds are relative to row0) -> out [3, H, W] per frame.  The fp32 value
// is the reference's, op by op: numpy's float32 x / 255, then torch's 2 * x and - 1 (no contraction into an FMA).
template <typename T>
__global__ void __launch_bounds__(128) resize_v_kernel(const uint8_t* __restrict__ src, long long src_frame, int row0,
                                                       const int2* __restrict__ bounds, const int* __restrict__ coeffs, int ksize,
                                                       T* __restrict__ out, int H, int W, int n) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int y = blockIdx.y;
    if (x >= W) return;
    const int2 b = __ldg(&bounds[y]);
    const int* k = coeffs + static_cast<long long>(y) * ksize;
    const long long plane = static_cast<long long>(H) * W;
    for (int f = blockIdx.z; f < n; f += gridDim.z) {
        const uint8_t* s = src + f * src_frame + (static_cast<long long>(b.x - row0) * W + x) * 3;
        int a[3] = {1 << (kPrecisionBits - 1), 1 << (kPrecisionBits - 1), 1 << (kPrecisionBits - 1)};
        for (int j = 0; j < b.y; ++j) {
            const int kj = __ldg(&k[j]);
            const uint8_t* p = s + static_cast<long long>(j) * W * 3;
            a[0] += p[0] * kj;
            a[1] += p[1] * kj;
            a[2] += p[2] * kj;
        }
        T* o = out + f * 3 * plane + static_cast<long long>(y) * W + x;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float u = static_cast<float>(clip8(a[c]));
            store(o + c * plane, __fsub_rn(__fmul_rn(2.0f, __fdiv_rn(u, 255.0f)), 1.0f));
        }
    }
}

dim3 grid_of(int width, int height, int n) { return dim3((width + 127) / 128, height, n < 65535 ? n : 65535); }

}  // namespace

int resize_table(int in_size, int out_size, int* ksize, int* bounds, int* coeffs) {
    if (in_size < 1 || out_size < 1 || in_size > kResizeMaxSize || out_size > kResizeMaxSize) return -1;
    const Table t = build_table(in_size, out_size);
    *ksize = t.ksize;
    if (bounds) std::copy(t.bounds.begin(), t.bounds.end(), bounds);
    if (coeffs) std::copy(t.coeffs.begin(), t.coeffs.end(), coeffs);
    return 0;
}

int frames_resize(const uint8_t* src, int n, int H0, int W0, void* out, int H, int W, int out_fp16, uint8_t* tmp,
                  cudaStream_t stream) {
    DeviceTable tv, th;
    int rc = device_table(H0, H, &tv);
    if (rc == 0 && W != W0) rc = device_table(W0, W, &th);
    if (rc != 0) return rc;
    const uint8_t* rows = src;
    long long rows_frame = static_cast<long long>(H0) * W0 * 3;
    int row0 = 0;
    if (W != W0) {
        const int nrows = tv.last - tv.first;
        resize_h_kernel<<<grid_of(W, nrows, n), 128, 0, stream>>>(src, rows_frame, W0, tv.first, nrows, th.bounds, th.coeffs,
                                                                   th.ksize, tmp, W, n);
        if ((rc = launch_status("frames_resize: horizontal pass")) != 0) return rc;
        rows = tmp;
        rows_frame = static_cast<long long>(nrows) * W * 3;
        row0 = tv.first;
    }
    if (out_fp16)
        resize_v_kernel<__half><<<grid_of(W, H, n), 128, 0, stream>>>(rows, rows_frame, row0, tv.bounds, tv.coeffs, tv.ksize,
                                                                       static_cast<__half*>(out), H, W, n);
    else
        resize_v_kernel<float><<<grid_of(W, H, n), 128, 0, stream>>>(rows, rows_frame, row0, tv.bounds, tv.coeffs, tv.ksize,
                                                                      static_cast<float*>(out), H, W, n);
    return launch_status("frames_resize: vertical pass");
}

}  // namespace t2v
