// GroupNorm (32 groups) statistics + apply(+SiLU), and LayerNorm, on channels-last fp16 token matrices.
// HBM-bound kernels: algorithmic bytes = 2 B/element read for stats, 2 B read + 2 B write for apply.
//
// Reduction domains (SURVEY.md appendix B): 4-D GroupNorm = one frame (h*w rows); 5-D GroupNorm = one sample
// (F*h*w rows).  Both are "instances" of `rows_per_inst` consecutive rows here.
// fp32 math throughout (the reference runs group_norm / layer_norm / SiLU-after-norm in fp32 under autocast and
// rounds to fp16 only when the value enters the next conv/linear -- exactly where these kernels round).
// GroupNorm statistics are summed as x - K_g in fp32, with a pivot K_g per (instance, group): the value of the group's first
// channel in the instance's first row.  Raw fp32 sums of x and x^2 would lose the variance to cancellation once
// |mean| / std reaches ~100 (E[x^2] - mean^2); shifted by a sample of the group, the sums stay of the size of the spread.
// The fold turns them back into raw moments in double (sum x = S + nK, sum x^2 = Q + 2KS + nK^2), where the cancellation
// of var = E[x^2] - mean^2 costs only (mean / std)^2 2^-53.
#include <algorithm>
#include <cstring>

#include "common.cuh"
#include "kernels.cuh"
#include "shard.cuh"

namespace t2v {

namespace {

constexpr int kGroups = 32;
constexpr int kNormThreads = 320;    // = 8 x 40 = 4 x 80 = 2 x 160 vectors: whole rows of C = 320 / 640 / 1280 per pass
constexpr int kMaxInst = 65535;             // instances (frames x samples) per call: gridDim.y
constexpr size_t kCounterBytes = 1 << 20;   // chunk counters [0, kMaxInst) | fused-kernel barrier generations from word 131072

// Thread mapping shared by the statistics and the apply kernel: a block covers RL = 320 / (C/8) consecutive rows per
// pass; thread (rl, vc) owns the 16-byte vector vc (8 channels) of rows rl, rl + RL, ...  Consecutive threads read
// consecutive 16 B, the channel identity of a thread never changes (per-channel accumulators / scale+shift live in
// registers), no integer division or shared-memory traffic in the streaming loop.
struct RowMap {
    int rl, vc, RL;
    bool active;
};
__device__ __forceinline__ RowMap row_map(int C8) {
    RowMap m;
    m.RL = kNormThreads / C8;
    m.rl = static_cast<int>(threadIdx.x) / C8;
    m.vc = static_cast<int>(threadIdx.x) - m.rl * C8;
    m.active = m.rl < m.RL;
    return m;
}

// The pivots K_g of the 8 channels a thread owns: x[first row of the instance, first channel of the channel's group].
__device__ __forceinline__ void load_pivots(const __half* inst_row0, int vc, int cpg, float (&k)[8]) {
#pragma unroll
    for (int e = 0; e < 8; ++e) k[e] = __half2float(inst_row0[(vc * 8 + e) / cpg * cpg]);
}

// Shifted per-thread sums of one 16-byte vector: s += x - K, q += (x - K)^2.
__device__ __forceinline__ void accum_vec(const uint4& v, const float (&k)[8], float (&s)[8], float (&q)[8]) {
    const __half2* h2 = reinterpret_cast<const __half2*>(&v);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h2[e]);
        const float d0 = f.x - k[2 * e], d1 = f.y - k[2 * e + 1];
        s[2 * e] += d0;
        q[2 * e] = fmaf(d0, d0, q[2 * e]);
        s[2 * e + 1] += d1;
        q[2 * e + 1] = fmaf(d1, d1, q[2 * e + 1]);
    }
}

// Raw moments (sum x, sum x^2) of a group from its shifted sums (S, Q) over n elements and its pivot K, in double.
__device__ __forceinline__ void unshift(double& a, double& b, double n, float K) {
    const double k = K;
    b += (2.0 * a + n * k) * k;
    a += n * k;
}

// partial[(inst * nchunks + chunk) * 32 + g] = (sum, sumsq) of x - K_g; the last block of an instance folds them (in
// chunk order, double precision) into stats[inst*32+g] = (mean, rstd) -> deterministic, no float atomics in HBM.
__global__ void __launch_bounds__(kNormThreads) gn_stats_kernel(const __half* __restrict__ x, long long ld, int C,
                                                                int rows_per_inst, int rows_per_chunk, int nchunks,
                                                                float eps, float2* __restrict__ partial,
                                                                unsigned int* __restrict__ counters,
                                                                float2* __restrict__ stats, const GnShard gs) {
    extern __shared__ float sm[];          // red[2][RL][C] | s_sum[C] | s_sq[C]
    __shared__ bool is_last;
    const int inst = blockIdx.y;
    const int chunk = blockIdx.x;
    const int C8 = C >> 3;
    const RowMap m = row_map(C8);
    float* red = sm;                        // [2][RL][C]
    float* s_sum = sm + 2 * m.RL * C;
    float* s_sq = s_sum + C;
    const int r0 = chunk * rows_per_chunk;
    const int r1 = min(r0 + rows_per_chunk, rows_per_inst);
    const __half* base = x + static_cast<long long>(inst) * rows_per_inst * ld;
    const int cpg = C / kGroups;
    float s[8], q[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) s[e] = q[e] = 0.f;
    if (m.active) {
        float k[8];
        load_pivots(base, m.vc, cpg, k);
        constexpr int U = 4;               // independent 16-byte loads in flight per thread
        const __half* p = base + static_cast<long long>(r0 + m.rl) * ld + m.vc * 8;
        const long long step = static_cast<long long>(m.RL) * ld;
        int r = r0 + m.rl;
        for (; r + (U - 1) * m.RL < r1; r += U * m.RL) {
            uint4 v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) v[u] = __ldg(reinterpret_cast<const uint4*>(p + u * step));
            p += U * step;
#pragma unroll
            for (int u = 0; u < U; ++u) accum_vec(v[u], k, s, q);
        }
        for (; r < r1; r += m.RL) {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
            p += step;
            accum_vec(v, k, s, q);
        }
        // cross-row-lane reduction through smem in a fixed order (no atomics: bit-reproducible run to run)
        float4* d0 = reinterpret_cast<float4*>(red + (0 * m.RL + m.rl) * C + m.vc * 8);
        float4* d1 = reinterpret_cast<float4*>(red + (1 * m.RL + m.rl) * C + m.vc * 8);
        d0[0] = make_float4(s[0], s[1], s[2], s[3]);
        d0[1] = make_float4(s[4], s[5], s[6], s[7]);
        d1[0] = make_float4(q[0], q[1], q[2], q[3]);
        d1[1] = make_float4(q[4], q[5], q[6], q[7]);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += kNormThreads) {
        float a = 0.f, b = 0.f;
        for (int y = 0; y < m.RL; ++y) {
            a += red[(0 * m.RL + y) * C + c];
            b += red[(1 * m.RL + y) * C + c];
        }
        s_sum[c] = a;
        s_sq[c] = b;
    }
    __syncthreads();
    if (threadIdx.x < kGroups) {
        float a = 0.f, b = 0.f;
        for (int c = 0; c < cpg; ++c) {
            a += s_sum[threadIdx.x * cpg + c];
            b += s_sq[threadIdx.x * cpg + c];
        }
        partial[(static_cast<long long>(inst) * nchunks + chunk) * kGroups + threadIdx.x] = make_float2(a, b);
    }
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned int prev = atomicAdd(&counters[inst], 1u);
        is_last = (prev == static_cast<unsigned int>(nchunks - 1));
    }
    __syncthreads();
    if (is_last) {
        __threadfence();
        // fold the chunk partials: 8 thread-parts per group read strided chunks (independent L2 loads in flight), then a
        // fixed-order combine -> deterministic and no serial chain of nchunks dependent loads
        __shared__ double fold[8][kGroups][2];
        if (threadIdx.x < 256) {
            const int gidx = threadIdx.x & 31, part = threadIdx.x >> 5;
            double a = 0.0, b = 0.0;
#pragma unroll 4
            for (int ch = part; ch < nchunks; ch += 8) {
                const float2 pp = __ldcg(&partial[(static_cast<long long>(inst) * nchunks + ch) * kGroups + gidx]);
                a += pp.x;
                b += pp.y;
            }
            fold[part][gidx][0] = a;
            fold[part][gidx][1] = b;
        }
        __syncthreads();
        if (threadIdx.x < kGroups) {
            double a = 0.0, b = 0.0;
#pragma unroll
            for (int part = 0; part < 8; ++part) {
                a += fold[part][threadIdx.x][0];
                b += fold[part][threadIdx.x][1];
            }
            double n = static_cast<double>(rows_per_inst) * cpg;
            unshift(a, b, n, __half2float(base[threadIdx.x * cpg]));
            if (gs.peers.nranks > 1) {
                // 5-D GroupNorm of a frame-sharded clip (pixel-sharded layout): this rank's (sum, sumsq) of the sample go to
                // every rank over NVLink peer stores; all ranks then fold the P contributions in rank order, so mean / rstd
                // are bit-identical everywhere.  threadIdx.x < 32 = warp 0 only.
                const int me = gs.peers.rank, nr = gs.peers.nranks;
                ShardComm* mine = gs.peers.comm[me];
                const unsigned int e = *reinterpret_cast<volatile unsigned int*>(&mine->epoch);
                for (int r = 0; r < nr; ++r) gs.peers.comm[r]->gn_part[gs.slot][inst][me][threadIdx.x] = make_double2(a, b);
                __threadfence_system();
                __syncwarp();
                if (static_cast<int>(threadIdx.x) < nr) {
                    st_release_sys(&gs.peers.comm[threadIdx.x]->gn_flag[gs.slot][inst][me], e);
                    spin_until_ge(&mine->gn_flag[gs.slot][inst][threadIdx.x], e);
                }
                __syncwarp();
                a = 0.0;
                b = 0.0;
                for (int r = 0; r < nr; ++r) {
                    const double2 v = __ldcv(&mine->gn_part[gs.slot][inst][r][threadIdx.x]);
                    a += v.x;
                    b += v.y;
                }
                n = static_cast<double>(gs.total_rows_per_inst) * cpg;
            }
            const double mean = a / n;
            double var = b / n - mean * mean;
            if (var < 0.0) var = 0.0;
            stats[inst * kGroups + threadIdx.x] =
                make_float2(static_cast<float>(mean), static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps))));
        }
        if (threadIdx.x == 0) counters[inst] = 0u;     // self-cleaning for the next launch
    }
}

// x * sigmoid(x) with one ex2 and one rcp on the MUFU (no IEEE division): the apply pass is MUFU-limited otherwise
__device__ __forceinline__ float silu_f(float v) {
    float e, r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(v * -1.4426950408889634f));
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
    return v * r;
}

// Per-channel scale a = rstd * gamma, mean and beta of the 8 channels a thread owns.
struct GnAffine {
    float a[8], mean[8], beta[8];
};
__device__ __forceinline__ void gn_affine(GnAffine& t, const float2* st, const __half* gamma, const __half* beta, int vc, int cpg) {
    const uint4 gv = __ldg(reinterpret_cast<const uint4*>(gamma + vc * 8));
    const uint4 bv = __ldg(reinterpret_cast<const uint4*>(beta + vc * 8));
    const __half* gh = reinterpret_cast<const __half*>(&gv);
    const __half* bh = reinterpret_cast<const __half*>(&bv);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
        const float2 ms = st[(vc * 8 + e) / cpg];
        t.mean[e] = ms.x;
        t.a[e] = ms.y * __half2float(gh[e]);
        t.beta[e] = __half2float(bh[e]);
    }
}

// y = act((x - mean) * a + beta): centring before the scale keeps a constant group at exactly beta, where
// x * a + (beta - mean * a) would leave the rounding of mean * a (|mean| / sqrt(eps) large) in the output.
template <bool SILU>
__device__ __forceinline__ uint4 gn_apply_vec(const uint4& v, const GnAffine& t) {
    const __half2* h2 = reinterpret_cast<const __half2*>(&v);
    uint4 o;
    __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(h2[e]);
        float u0 = fmaf(f.x - t.mean[2 * e], t.a[2 * e], t.beta[2 * e]);
        float u1 = fmaf(f.y - t.mean[2 * e + 1], t.a[2 * e + 1], t.beta[2 * e + 1]);
        if (SILU) {
            u0 = silu_f(u0);
            u1 = silu_f(u1);
        }
        oh[e] = __floats2half2_rn(u0, u1);
    }
    return o;
}

// grid = (row blocks, instances).  Each thread folds (rstd, gamma) of ITS 8 channels into scale registers, then streams
// its rows: y = act((x - mean[c]) * a[c] + beta[c]) -- one FADD and one FMA (+ SiLU) per element, 16-byte accesses.
template <bool SILU>
__global__ void __launch_bounds__(kNormThreads) gn_apply_kernel(const __half* __restrict__ x, long long ldx,
                                                                __half* __restrict__ y, long long ldy, int C,
                                                                int rows_per_inst, int rows_per_block,
                                                                const float2* __restrict__ stats,
                                                                const __half* __restrict__ gamma,
                                                                const __half* __restrict__ beta) {
    const int inst = blockIdx.y;
    const int C8 = C >> 3;
    const int cpg = C / kGroups;
    const RowMap m = row_map(C8);
    if (!m.active) return;
    GnAffine t;
    gn_affine(t, stats + inst * kGroups, gamma, beta, m.vc, cpg);
    const int r0 = blockIdx.x * rows_per_block;
    const int r1 = min(r0 + rows_per_block, rows_per_inst);
    const long long row0 = static_cast<long long>(inst) * rows_per_inst + r0 + m.rl;
    const __half* px = x + row0 * ldx + m.vc * 8;
    __half* py = y + row0 * ldy + m.vc * 8;
    const long long sx = static_cast<long long>(m.RL) * ldx, sy = static_cast<long long>(m.RL) * ldy;
    constexpr int U = 4;                   // independent 16-byte loads in flight per thread
    int r = r0 + m.rl;
    for (; r + (U - 1) * m.RL < r1; r += U * m.RL) {
        uint4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) v[u] = __ldg(reinterpret_cast<const uint4*>(px + u * sx));
        px += U * sx;
#pragma unroll
        for (int u = 0; u < U; ++u) *reinterpret_cast<uint4*>(py + u * sy) = gn_apply_vec<SILU>(v[u], t);
        py += U * sy;
    }
    for (; r < r1; r += m.RL) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(px));
        px += sx;
        *reinterpret_cast<uint4*>(py) = gn_apply_vec<SILU>(v, t);
        py += sy;
    }
}


// ---- single-launch GroupNorm: statistics -> per-instance barrier -> normalise (+SiLU) in ONE kernel.
// grid = (cpi, instances): the `cpi` CTAs of an instance are all co-resident (the host sizes the grid to the machine: no
// other kernel shares the SMs, every launch of the library is stream-ordered), so they can meet at a sense-reversing barrier
// in global memory.  When a CTA's row slice fits in shared memory it is kept there between the two passes: the activation
// is then read ONCE (2 B/elt read + 2 B/elt write instead of 4 + 2) and the second launch with its drain/fill bubble is gone.
// Deterministic: partials are folded in chunk order in double precision by every CTA of the instance.
template <bool SILU>
__global__ void __launch_bounds__(kNormThreads) gn_fused_kernel(const __half* __restrict__ x, long long ldx,
                                                                __half* __restrict__ y, long long ldy, int C,
                                                                int rows_per_inst, int rows_per_cta, float eps,
                                                                float2* __restrict__ partial, unsigned int* __restrict__ count,
                                                                unsigned int* __restrict__ gen, const __half* __restrict__ gamma,
                                                                const __half* __restrict__ beta, int cache) {
    extern __shared__ __align__(16) float sm[];   // red[2][RL][C] | s_sum[C] | s_sq[C] | fold[8][32][2] doubles | stats[32] float2 | slice
    const int inst = blockIdx.y;
    const int chunk = blockIdx.x;
    const int cpi = gridDim.x;
    const int C8 = C >> 3;
    const int cpg = C / kGroups;
    const RowMap m = row_map(C8);
    float* red = sm;
    float* s_sum = sm + 2 * m.RL * C;
    float* s_sq = s_sum + C;
    double* fold = reinterpret_cast<double*>(s_sq + C);                 // 8 * 32 * 2 doubles (offset is a multiple of 8 B: C % 8 == 0)
    float2* st = reinterpret_cast<float2*>(fold + 8 * kGroups * 2);
    uint4* slice = reinterpret_cast<uint4*>(st + kGroups);              // [rows_per_cta][C8] when `cache`
    const int r0 = chunk * rows_per_cta;
    const int r1 = min(r0 + rows_per_cta, rows_per_inst);
    const __half* base = x + static_cast<long long>(inst) * rows_per_inst * ldx;
    float s[8], q[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) s[e] = q[e] = 0.f;
    if (m.active) {
        float k[8];
        load_pivots(base, m.vc, cpg, k);
        constexpr int U = 4;
        const __half* p = base + static_cast<long long>(r0 + m.rl) * ldx + m.vc * 8;
        const long long step = static_cast<long long>(m.RL) * ldx;
        int r = r0 + m.rl;
        for (; r + (U - 1) * m.RL < r1; r += U * m.RL) {
            uint4 v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) v[u] = __ldg(reinterpret_cast<const uint4*>(p + u * step));
            p += U * step;
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if (cache) slice[static_cast<size_t>(r - r0 + u * m.RL) * C8 + m.vc] = v[u];
                accum_vec(v[u], k, s, q);
            }
        }
        for (; r < r1; r += m.RL) {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
            p += step;
            if (cache) slice[static_cast<size_t>(r - r0) * C8 + m.vc] = v;
            accum_vec(v, k, s, q);
        }
        float4* d0 = reinterpret_cast<float4*>(red + (0 * m.RL + m.rl) * C + m.vc * 8);
        float4* d1 = reinterpret_cast<float4*>(red + (1 * m.RL + m.rl) * C + m.vc * 8);
        d0[0] = make_float4(s[0], s[1], s[2], s[3]);
        d0[1] = make_float4(s[4], s[5], s[6], s[7]);
        d1[0] = make_float4(q[0], q[1], q[2], q[3]);
        d1[1] = make_float4(q[4], q[5], q[6], q[7]);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += kNormThreads) {
        float a = 0.f, b = 0.f;
        for (int yy = 0; yy < m.RL; ++yy) {
            a += red[(0 * m.RL + yy) * C + c];
            b += red[(1 * m.RL + yy) * C + c];
        }
        s_sum[c] = a;
        s_sq[c] = b;
    }
    __syncthreads();
    if (threadIdx.x < kGroups) {
        float a = 0.f, b = 0.f;
        for (int c = 0; c < cpg; ++c) {
            a += s_sum[threadIdx.x * cpg + c];
            b += s_sq[threadIdx.x * cpg + c];
        }
        partial[(static_cast<long long>(inst) * cpi + chunk) * kGroups + threadIdx.x] = make_float2(a, b);
    }
    if (cpi > 1) {
        // sense-reversing barrier over the CTAs of this instance: every CTA reads the generation BEFORE it arrives; the last
        // arriver resets the count and bumps the generation.  Bounded spin: a scheduling assumption that ever failed traps
        // instead of hanging the device.
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned int g0;
            asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(g0) : "l"(gen + inst) : "memory");
            __threadfence();
            const unsigned int prev = atomicAdd(&count[inst], 1u);
            if (prev == static_cast<unsigned int>(cpi - 1)) {
                count[inst] = 0u;
                __threadfence();
                asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(gen + inst), "r"(g0 + 1u) : "memory");
            } else {
                unsigned int g = g0;
                for (unsigned int spins = 0; g == g0; ++spins) {
                    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(g) : "l"(gen + inst) : "memory");
                    if (g == g0) {
                        __nanosleep(32);
                        if (spins > (1u << 25)) __trap();
                    }
                }
            }
        }
        __syncthreads();
    } else {
        __syncthreads();
    }
    if (threadIdx.x < 256) {
        const int gidx = threadIdx.x & 31, part = threadIdx.x >> 5;
        double a = 0.0, b = 0.0;
#pragma unroll 4
        for (int ch = part; ch < cpi; ch += 8) {
            const float2 pp = __ldcg(&partial[(static_cast<long long>(inst) * cpi + ch) * kGroups + gidx]);
            a += pp.x;
            b += pp.y;
        }
        fold[(part * kGroups + gidx) * 2 + 0] = a;
        fold[(part * kGroups + gidx) * 2 + 1] = b;
    }
    __syncthreads();
    if (threadIdx.x < kGroups) {
        double a = 0.0, b = 0.0;
#pragma unroll
        for (int part = 0; part < 8; ++part) {
            a += fold[(part * kGroups + threadIdx.x) * 2 + 0];
            b += fold[(part * kGroups + threadIdx.x) * 2 + 1];
        }
        const double n = static_cast<double>(rows_per_inst) * cpg;
        unshift(a, b, n, __half2float(base[threadIdx.x * cpg]));
        const double mean = a / n;
        double var = b / n - mean * mean;
        if (var < 0.0) var = 0.0;
        st[threadIdx.x] = make_float2(static_cast<float>(mean), static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps))));
    }
    __syncthreads();
    if (!m.active) return;
    GnAffine t;
    gn_affine(t, st, gamma, beta, m.vc, cpg);
    const long long row0 = static_cast<long long>(inst) * rows_per_inst + r0 + m.rl;
    const __half* px = x + row0 * ldx + m.vc * 8;
    __half* py = y + row0 * ldy + m.vc * 8;
    const long long sx = static_cast<long long>(m.RL) * ldx, sy = static_cast<long long>(m.RL) * ldy;
    constexpr int U = 4;
    int r = r0 + m.rl;
    for (; r + (U - 1) * m.RL < r1; r += U * m.RL) {
        uint4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u)
            v[u] = cache ? slice[static_cast<size_t>(r - r0 + u * m.RL) * C8 + m.vc] : __ldg(reinterpret_cast<const uint4*>(px + u * sx));
        px += U * sx;
#pragma unroll
        for (int u = 0; u < U; ++u) *reinterpret_cast<uint4*>(py + u * sy) = gn_apply_vec<SILU>(v[u], t);
        py += U * sy;
    }
    for (; r < r1; r += m.RL) {
        const uint4 v = cache ? slice[static_cast<size_t>(r - r0) * C8 + m.vc] : __ldg(reinterpret_cast<const uint4*>(px));
        px += sx;
        *reinterpret_cast<uint4*>(py) = gn_apply_vec<SILU>(v, t);
        py += sy;
    }
}

// one warp per row; C <= 2048, C % 8 == 0
__global__ void __launch_bounds__(256) layernorm_kernel(const __half* __restrict__ x, long long ldx,
                                                        __half* __restrict__ y, long long ldy, long long rows, int C,
                                                        const __half* __restrict__ gamma,
                                                        const __half* __restrict__ beta, float eps) {
    const int lane = threadIdx.x & 31;
    const long long row = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
    if (row >= rows) return;
    const int C8 = C >> 3;
    constexpr int MAXV = 8;
    uint4 v[MAXV];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
        const int vc = lane + k * 32;
        if (vc < C8) {
            v[k] = __ldg(reinterpret_cast<const uint4*>(x + row * ldx + vc * 8));
            const __half2* h2 = reinterpret_cast<const __half2*>(&v[k]);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 f = __half22float2(h2[e]);
                s += f.x + f.y;
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    const float mean = s / C;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
        const int vc = lane + k * 32;
        if (vc < C8) {
            const __half2* h2 = reinterpret_cast<const __half2*>(&v[k]);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 f = __half22float2(h2[e]);
                q += (f.x - mean) * (f.x - mean) + (f.y - mean) * (f.y - mean);
            }
        }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
    const float rstd = rsqrtf(q / C + eps);
#pragma unroll
    for (int k = 0; k < MAXV; ++k) {
        const int vc = lane + k * 32;
        if (vc < C8) {
            const uint4 gv = __ldg(reinterpret_cast<const uint4*>(gamma + vc * 8));
            const uint4 bv = __ldg(reinterpret_cast<const uint4*>(beta + vc * 8));
            const __half* xh = reinterpret_cast<const __half*>(&v[k]);
            const __half* gh = reinterpret_cast<const __half*>(&gv);
            const __half* bh = reinterpret_cast<const __half*>(&bv);
            uint4 o;
            __half* oh = reinterpret_cast<__half*>(&o);
#pragma unroll
            for (int e = 0; e < 8; ++e)
                oh[e] = __float2half_rn((__half2float(xh[e]) - mean) * rstd * __half2float(gh[e]) + __half2float(bh[e]));
            *reinterpret_cast<uint4*>(y + row * ldy + vc * 8) = o;
        }
    }
}

// (mean, rstd) per row; one warp per row, two rows in flight per warp, grid-stride over rows (a few resident blocks
// per SM instead of one short-lived block per 8 rows).  NV = ceil(C / 256) 16-byte vectors per lane.
template <int NV>
__global__ void __launch_bounds__(256) ln_rowstats_kernel(const __half* __restrict__ x, long long ldx, long long rows, int C,
                                                          float eps, float2* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const int C8 = C >> 3;
    const float inv_c = 1.0f / static_cast<float>(C);
    const long long wstride = static_cast<long long>(gridDim.x) * (blockDim.x >> 5);
    long long row = blockIdx.x * static_cast<long long>(blockDim.x >> 5) + (threadIdx.x >> 5);
    for (; row < rows; row += 2 * wstride) {
        const long long rowb = row + wstride;
        const bool hb = rowb < rows;
        uint4 va[NV], vb[NV];
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const int vc = lane + k * 32;
            va[k] = make_uint4(0u, 0u, 0u, 0u);
            vb[k] = make_uint4(0u, 0u, 0u, 0u);
            if (vc < C8) {
                va[k] = __ldg(reinterpret_cast<const uint4*>(x + row * ldx + vc * 8));
                if (hb) vb[k] = __ldg(reinterpret_cast<const uint4*>(x + rowb * ldx + vc * 8));
            }
        }
        float sa = 0.f, sb = 0.f;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            const __half2* ha = reinterpret_cast<const __half2*>(&va[k]);
            const __half2* hbp = reinterpret_cast<const __half2*>(&vb[k]);
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float2 fa = __half22float2(ha[e]);
                const float2 fb = __half22float2(hbp[e]);
                sa += fa.x + fa.y;
                sb += fb.x + fb.y;
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            sa += __shfl_xor_sync(0xffffffffu, sa, o);
            sb += __shfl_xor_sync(0xffffffffu, sb, o);
        }
        const float ma = sa * inv_c, mb = sb * inv_c;
        float qa = 0.f, qb = 0.f;
#pragma unroll
        for (int k = 0; k < NV; ++k) {
            if (lane + k * 32 < C8) {          // padding vectors are zero, not (0 - mean)
                const __half2* ha = reinterpret_cast<const __half2*>(&va[k]);
                const __half2* hbp = reinterpret_cast<const __half2*>(&vb[k]);
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const float2 fa = __half22float2(ha[e]);
                    const float2 fb = __half22float2(hbp[e]);
                    qa += (fa.x - ma) * (fa.x - ma) + (fa.y - ma) * (fa.y - ma);
                    qb += (fb.x - mb) * (fb.x - mb) + (fb.y - mb) * (fb.y - mb);
                }
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            qa += __shfl_xor_sync(0xffffffffu, qa, o);
            qb += __shfl_xor_sync(0xffffffffu, qb, o);
        }
        if (lane == 0) {
            out[row] = make_float2(ma, rsqrtf(qa * inv_c + eps));
            if (hb) out[rowb] = make_float2(mb, rsqrtf(qb * inv_c + eps));
        }
    }
}

}  // namespace

static size_t stats_smem_bytes(int C) {
    const int RL = kNormThreads / (C / 8);
    return static_cast<size_t>(2 * RL * C + 2 * C) * sizeof(float);
}

int gn_rows_per_chunk(int rows_per_inst, int n_inst, int num_sms) {
    // ~2 blocks per SM: fat blocks amortise the per-block latency chain (few dependent loads per thread otherwise)
    long long want = static_cast<long long>(num_sms) * 2;
    long long chunks_per_inst = (want + n_inst - 1) / n_inst;
    if (chunks_per_inst < 1) chunks_per_inst = 1;
    long long rpc = (rows_per_inst + chunks_per_inst - 1) / chunks_per_inst;
    if (rpc < 8) rpc = 8;
    rpc = (rpc + 7) / 8 * 8;
    return static_cast<int>(rpc);
}

size_t gn_workspace_bytes(int rows_per_inst, int n_inst, int num_sms) {
    const int rpc = gn_rows_per_chunk(rows_per_inst, n_inst, num_sms);
    const int nchunks = (rows_per_inst + rpc - 1) / rpc;
    // counters (fixed-size region at the START: their location must not depend on the call's shape, they have to
    // stay zero between launches) + stats + partials
    // (+ the single-launch kernel's partials: up to 2 CTAs per SM in total)
    return kCounterBytes + static_cast<size_t>(n_inst) * kGroups * sizeof(float2) +
           static_cast<size_t>(n_inst) * nchunks * kGroups * sizeof(float2) +
           (static_cast<size_t>(2 * num_sms) + n_inst) * kGroups * sizeof(float2) + 256;
}

static bool misaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }

int groupnorm_check(const __half* x, long long ldx, const __half* y, long long ldy, long long rows, int C, int rows_per_inst,
                    const __half* gamma, const __half* beta) {
    if (C <= 0 || C % 32 != 0 || C / 8 > kNormThreads) {
        set_error("groupnorm: C = %d must be a positive multiple of 32, at most %d", C, 8 * kNormThreads);
        return -1;
    }
    if (rows_per_inst <= 0 || rows < rows_per_inst || rows % rows_per_inst != 0 || rows / rows_per_inst > kMaxInst) {
        set_error("groupnorm: rows = %lld must be 1 to %d whole instances of rows_per_inst = %d", rows, kMaxInst, rows_per_inst);
        return -1;
    }
    // 16-byte vector loads and stores of x, y, gamma and beta
    if (ldx < C || ldy < C || (ldx & 7) != 0 || (ldy & 7) != 0 || misaligned16(x) || misaligned16(y) || misaligned16(gamma) ||
        misaligned16(beta)) {
        set_error("groupnorm: x, y, gamma, beta must be 16-byte aligned and ldx = %lld, ldy = %lld multiples of 8, >= C = %d", ldx,
                  ldy, C);
        return -1;
    }
    return 0;
}

float2* gn_workspace_stats(void* workspace) { return reinterpret_cast<float2*>(reinterpret_cast<uint8_t*>(workspace) + kCounterBytes); }

// the fused kernel's CTAs of one instance meet at a barrier: only launch it when the whole grid fits on the machine at once
static bool gn_fused_coresident(int silu, size_t smem, long long ctas, int num_sms) {
    int per_sm = 0;
    const cudaError_t e = silu ? cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gn_fused_kernel<true>, kNormThreads, smem)
                               : cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, gn_fused_kernel<false>, kNormThreads, smem);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return false;
    }
    return static_cast<long long>(per_sm) * num_sms >= ctas;
}

int groupnorm_silu(const __half* x, long long ldx, __half* y, long long ldy, long long rows, int C, int rows_per_inst,
                   const __half* gamma, const __half* beta, float eps, int silu, void* workspace, int num_sms,
                   cudaStream_t stream, int phase, const GnShard* shard) {
    if (groupnorm_check(x, ldx, y, ldy, rows, C, rows_per_inst, gamma, beta) != 0) return -1;
    const int n_inst = static_cast<int>(rows / rows_per_inst);
    const int rpc = gn_rows_per_chunk(rows_per_inst, n_inst, num_sms);
    const int nchunks = (rows_per_inst + rpc - 1) / rpc;
    uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
    unsigned int* counters = reinterpret_cast<unsigned int*>(ws);
    float2* stats = reinterpret_cast<float2*>(ws + kCounterBytes);
    float2* partial = stats + static_cast<size_t>(n_inst) * kGroups;
    // ---- single-launch path (phase 0, no cross-rank statistics): all CTAs of the grid must be co-resident
    if (phase == 0 && (shard == nullptr || shard->peers.nranks <= 1)) {
        const size_t inst_bytes = static_cast<size_t>(rows_per_inst) * C * sizeof(__half);
        const size_t fixed = stats_smem_bytes(C) + 8 * kGroups * 2 * sizeof(double) + kGroups * sizeof(float2);
        const size_t cache_cap = 200 * 1024 - fixed;                     // slice bytes a lone CTA per SM can keep
        const int RL = kNormThreads / (C / 8);
        int cpi = 0, cache = 0;
        if (n_inst <= num_sms) {
            const int cmax = num_sms / n_inst;                              // one CTA per SM when caching
            const long long need = (static_cast<long long>(inst_bytes) + cache_cap - 1) / static_cast<long long>(cache_cap);
            if (need <= cmax) {
                cpi = cmax;
                cache = 1;
            }
        }
        if (!cache && n_inst <= 2 * num_sms && fixed <= 100 * 1024) cpi = (2 * num_sms) / n_inst;      // two lean CTAs per SM, second pass from L2
        if (cpi > 0) {
            const int max_useful = (rows_per_inst + RL - 1) / RL;            // at least one row pass per CTA
            if (cpi > max_useful) cpi = max_useful;
            if (cpi < 1) cpi = 1;
            int rpc2 = (rows_per_inst + cpi - 1) / cpi;
            cpi = (rows_per_inst + rpc2 - 1) / rpc2;
            size_t smem = fixed + (cache ? static_cast<size_t>(rpc2) * C * sizeof(__half) : 0);
            if (cache && smem > 226 * 1024) {
                cache = 0;
                smem = fixed;
            }
            static bool attr_done = false;
            if (!attr_done) {
                cudaFuncSetAttribute(gn_fused_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
                cudaFuncSetAttribute(gn_fused_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024);
                attr_done = true;
            }
            // a grid that cannot be co-resident would spin at the barrier: it takes the two kernels below instead
            if (gn_fused_coresident(silu, smem, static_cast<long long>(cpi) * n_inst, num_sms)) {
                unsigned int* gen = counters + (kCounterBytes / sizeof(unsigned int)) / 2;
                if (silu)
                    gn_fused_kernel<true><<<dim3(cpi, n_inst), kNormThreads, smem, stream>>>(x, ldx, y, ldy, C, rows_per_inst, rpc2, eps,
                                                                                             partial, counters, gen, gamma, beta, cache);
                else
                    gn_fused_kernel<false><<<dim3(cpi, n_inst), kNormThreads, smem, stream>>>(x, ldx, y, ldy, C, rows_per_inst, rpc2,
                                                                                              eps, partial, counters, gen, gamma, beta,
                                                                                              cache);
                return launch_status("norm launch");
            }
        }
    }
    GnShard gs;
    memset(&gs, 0, sizeof(gs));
    if (shard != nullptr && shard->peers.nranks > 1) {
        if (n_inst > SHARD_MAX_INST || shard->slot < 0 || shard->slot >= SHARD_MAX_GN) return -4;
        gs = *shard;
    }
    if (phase != 2)
        gn_stats_kernel<<<dim3(nchunks, n_inst), kNormThreads, stats_smem_bytes(C), stream>>>(x, ldx, C, rows_per_inst,
                                                                                              rpc, nchunks, eps, partial, counters, stats, gs);
    if (phase == 1) return launch_status("norm launch");
    // rows per apply block: ~4 blocks per SM overall, at least 4 rows
    long long want_blocks = static_cast<long long>(num_sms) * 4;
    long long per_inst = (want_blocks + n_inst - 1) / n_inst;
    if (per_inst < 1) per_inst = 1;
    long long rpb = (rows_per_inst + per_inst - 1) / per_inst;
    if (rpb < 4) rpb = 4;
    const int nblk = static_cast<int>((rows_per_inst + rpb - 1) / rpb);
    if (silu)
        gn_apply_kernel<true><<<dim3(nblk, n_inst), kNormThreads, 0, stream>>>(x, ldx, y, ldy, C, rows_per_inst,
                                                                               static_cast<int>(rpb), stats, gamma, beta);
    else
        gn_apply_kernel<false><<<dim3(nblk, n_inst), kNormThreads, 0, stream>>>(x, ldx, y, ldy, C, rows_per_inst,
                                                                                static_cast<int>(rpb), stats, gamma, beta);
    return launch_status("norm launch");
}

int layernorm_rowstats(const __half* x, long long ldx, long long rows, int C, float eps, float2* out, cudaStream_t stream) {
    if (C % 8 != 0 || C > 2048) return -1;
    const long long need = (rows + 15) / 16;                           // 8 warps x 2 rows per block pass
    const unsigned int grid = static_cast<unsigned int>(std::min<long long>(need, static_cast<long long>(num_sms()) * 8));
    const int nv = (C / 8 + 31) / 32;
    if (nv <= 2) ln_rowstats_kernel<2><<<grid, 256, 0, stream>>>(x, ldx, rows, C, eps, out);
    else if (nv <= 3) ln_rowstats_kernel<3><<<grid, 256, 0, stream>>>(x, ldx, rows, C, eps, out);
    else if (nv <= 5) ln_rowstats_kernel<5><<<grid, 256, 0, stream>>>(x, ldx, rows, C, eps, out);
    else ln_rowstats_kernel<8><<<grid, 256, 0, stream>>>(x, ldx, rows, C, eps, out);
    return launch_status("norm launch");
}

int layernorm(const __half* x, long long ldx, __half* y, long long ldy, long long rows, int C, const __half* gamma,
              const __half* beta, float eps, cudaStream_t stream) {
    if (C <= 0 || C % 8 != 0 || C > 2048 || rows < 1 || rows >= (1LL << 31)) {
        set_error("layernorm: C = %d must be a multiple of 8 from 8 to 2048 and rows = %lld from 1 to 2^31 - 1", C, rows);
        return -1;
    }
    // 16-byte vector loads and stores of x, y, gamma and beta
    if (ldx < C || ldy < C || (ldx & 7) != 0 || (ldy & 7) != 0 || misaligned16(x) || misaligned16(y) || misaligned16(gamma) ||
        misaligned16(beta)) {
        set_error("layernorm: x, y, gamma, beta must be 16-byte aligned and ldx = %lld, ldy = %lld multiples of 8, >= C = %d", ldx,
                  ldy, C);
        return -1;
    }
    const long long blocks = (rows + 7) / 8;
    layernorm_kernel<<<static_cast<unsigned int>(blocks), 256, 0, stream>>>(x, ldx, y, ldy, rows, C, gamma, beta, eps);
    return launch_status("norm launch");
}

}  // namespace t2v
