// Spatial self-attention on the Hopper tensor cores (wgmma): softmax(Q K^T * scale) V, head_dim 64, long sequences
// (S = h*w tokens of one frame, t2v_model.py:540-584 with the (b, hw, c) token layout of :639-658).
//
// One CTA owns 128 queries of one (frame, head) and streams the keys/values in 128-row tiles:
//
//   warpgroup 0      TMA producer   Q (16 KB, once), then K_j / V_j tiles into a 4-stage ring -- straight out of the fused
//                                   [tokens, 3C] QKV matrix: the head is a column offset of the tensor map, rows past the
//                                   end of the frame are TMA zero fill.
//   warpgroups 1, 2  consumers      64 query rows each:
//                                   S  = Q K_j^T   4 x wgmma m64n128k16, both operands from shared memory, fp32 in registers
//                                   online softmax on the accumulator fragment (row max / sum across the 4 threads of a row)
//                                   O += P V_j     8 x wgmma m64n64k16: A = P as fp16 register fragments (the S accumulator
//                                                  layout IS the A-fragment layout, no shared-memory round trip), B = V_j as
//                                                  it lies in the token matrix ([key][d] rows) through an MN-major descriptor
//                                                  -- no transposed copy of V.
//   setmaxnreg moves registers from the producer warpgroup to the consumers.
//
// Both consumer warpgroups share every K/V tile (one L2 read per 128 queries).
//
// attention() (attention.cu) routes here the calls attention_tc_eligible accepts; attention_tc encodes the three tensor
// maps and launches.
//
// Numerics (= torch SDPA fused kernels the reference dispatches to, t2v_model.py:561-569): fp16 operands, fp32 scores,
// fp32 online softmax with the scale folded into exp2, P rounded to fp16 for P.V, fp32 output accumulation,
// normalised by the fp32 row sum at the end.
#include <cuda.h>

#include <cstdio>

#include "gemm_tc.cuh"
#include "common.cuh"
#include "kernels.cuh"
#include "ptx.cuh"

namespace t2v {

namespace {

constexpr int HD = 64;
constexpr int BQ = 128;                 // query rows per CTA (64 per consumer warpgroup)
constexpr int BKV = 128;                // keys per iteration
constexpr int ST = 4;                   // K/V ring stages
constexpr int TILE_BYTES = 128 * 128;   // 128 rows x 64 fp16
constexpr int SMEM_Q = 0;
constexpr int SMEM_K = SMEM_Q + TILE_BYTES;
constexpr int SMEM_V = SMEM_K + ST * TILE_BYTES;
constexpr int SMEM_BAR = SMEM_V + ST * TILE_BYTES;
constexpr int SMEM_TOTAL = SMEM_BAR + 256 + 1024;          // + alignment slack
constexpr int NTHREADS = 384;           // warpgroups: TMA | consumer rows 0-63 | consumer rows 64-127
constexpr int REGS_CONSUMER = 232;      // 2 x 128 x 232 + 128 x 40 <= 64 K
constexpr int REGS_PRODUCER = 40;

struct Args {
    __half* o;
    long long o_bs, o_ss;
    int sq, skv, kv_batch_div, n_kv;
    float sl2;                          // scale * log2(e)
};

__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
    const __half2 h = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&h);
}

__global__ void __launch_bounds__(NTHREADS, 1)
attention_tc_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_k,
                    const __grid_constant__ CUtensorMap map_v, const Args a) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + SMEM_BAR);
    uint64_t* bar_q = bars;                    // Q tile landed
    uint64_t* kv_full = bars + 1;              // [ST] K_j, V_j landed
    uint64_t* kv_empty = kv_full + ST;         // [ST] both consumer warpgroups are done with the stage

    const int wg = threadIdx.x >> 7;
    const int q0 = blockIdx.x * BQ;
    const int head = blockIdx.y;
    const int b = blockIdx.z;
    const int n_kv = a.n_kv;

    if (threadIdx.x == 0) {
        mbar_init(bar_q, 1);
        for (int s = 0; s < ST; ++s) {
            mbar_init(&kv_full[s], 1);
            mbar_init(&kv_empty[s], 2);
        }
        fence_barrier_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ------------------------------------------------------------------ TMA producer
        setmaxnreg_dec<REGS_PRODUCER>();
        if (threadIdx.x < 32 && elect_one()) {
            tma_prefetch_desc(&map_q);
            tma_prefetch_desc(&map_k);
            tma_prefetch_desc(&map_v);
            mbar_expect_tx(bar_q, TILE_BYTES);
            tma_load_3d(smem + SMEM_Q, &map_q, bar_q, head * HD, q0, b);
            const int bkv = b / a.kv_batch_div;
            for (int j = 0; j < n_kv; ++j) {
                const int s = j % ST;
                if (j >= ST) mbar_wait(&kv_empty[s], ((j / ST) - 1) & 1);
                mbar_expect_tx(&kv_full[s], 2 * TILE_BYTES);
                tma_load_3d(smem + SMEM_K + s * TILE_BYTES, &map_k, &kv_full[s], head * HD, j * BKV, bkv);
                tma_load_3d(smem + SMEM_V + s * TILE_BYTES, &map_v, &kv_full[s], head * HD, j * BKV, bkv);
            }
        }
        __syncwarp();
    } else {
        // ------------------------------------------------------------------ consumers (64 query rows each)
        setmaxnreg_inc<REGS_CONSUMER>();
        const int cw = wg - 1;
        const int lt = threadIdx.x & 127;
        const int wr = lt >> 5, lane = lt & 31;
        const int quad = lane & 3;
        const float sl2 = a.sl2;
        const uint64_t dq = wgmma_desc_sw128(smem_u32(smem + SMEM_Q) + cw * (64 * 128));
        const uint32_t sk_addr = smem_u32(smem + SMEM_K);
        const uint32_t sv_addr = smem_u32(smem + SMEM_V);
        float o[HD / 2];
#pragma unroll
        for (int i = 0; i < HD / 2; ++i) o[i] = 0.f;
        float m_run[2] = {-INFINITY, -INFINITY};      // running max of rows g, g + 8 (g = lane / 4)
        float l_run[2] = {0.f, 0.f};                  // this thread's share of the row sums
        mbar_wait(bar_q, 0);

        for (int j = 0; j < n_kv; ++j) {
            const int s = j % ST;
            mbar_wait(&kv_full[s], (j / ST) & 1);
            float sc[BKV / 2];
            const uint64_t dk = wgmma_desc_sw128(sk_addr + s * TILE_BYTES);
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < HD / 16; ++ks) wgmma_ss<BKV>(sc, dq + 2 * ks, dk + 2 * ks, ks > 0 ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int i = 0; i < BKV / 2; ++i) reg_fence(sc[i]);

            // ---- padding keys of a ragged last tile -> -inf; row max over the quad's 4 threads
            const int valid = a.skv - j * BKV;
            if (valid < BKV) {
#pragma unroll
                for (int i = 0; i < BKV / 2; ++i)
                    if (8 * (i >> 2) + 2 * quad + (i & 1) >= valid) sc[i] = -INFINITY;
            }
            float corr[2], msc[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                float mx = -INFINITY;
#pragma unroll
                for (int jj = 0; jj < BKV / 8; ++jj) mx = fmaxf(mx, fmaxf(sc[4 * jj + 2 * h], sc[4 * jj + 2 * h + 1]));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                const float m_new = fmaxf(m_run[h], mx);
                corr[h] = ex2_approx((m_run[h] - m_new) * sl2);         // exp2(-inf) = 0 on the first tile
                m_run[h] = m_new;
                msc[h] = m_new * sl2;
                l_run[h] *= corr[h];
            }
#pragma unroll
            for (int i = 0; i < HD / 2; ++i) o[i] *= corr[(i >> 1) & 1];

            // ---- P = exp2(S * c - m * c) -> fp16 A fragments (k-step ks covers keys 16 ks .. 16 ks + 15)
            uint32_t pf[BKV / 16][4];
#pragma unroll
            for (int ks = 0; ks < BKV / 16; ++ks) {
                float pv[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                    const int h = (e >> 1) & 1;
                    pv[e] = ex2_approx(fmaf(sc[8 * ks + e], sl2, -msc[h]));     // exp2(-inf) = 0
                    l_run[h] += pv[e];
                }
                pf[ks][0] = pack_half2(pv[0], pv[1]);      // row g,     keys 16 ks + 2 quad + {0, 1}
                pf[ks][1] = pack_half2(pv[2], pv[3]);      // row g + 8, same keys
                pf[ks][2] = pack_half2(pv[4], pv[5]);      // row g,     keys 16 ks + 8 + 2 quad + {0, 1}
                pf[ks][3] = pack_half2(pv[6], pv[7]);      // row g + 8, same keys
            }
            // ---- O += P V_j: 16 key rows of V = 2048 B per k-step
#pragma unroll
            for (int i = 0; i < HD / 2; ++i) reg_fence(o[i]);
            wgmma_fence();
#pragma unroll
            for (int ks = 0; ks < BKV / 16; ++ks)
                wgmma_rs_n64_tb(o, pf[ks], wgmma_desc_sw128(sv_addr + s * TILE_BYTES + ks * 2048));
            wgmma_commit();
            wgmma_wait<0>();
#pragma unroll
            for (int i = 0; i < HD / 2; ++i) reg_fence(o[i]);
            if (lt == 0) mbar_arrive(&kv_empty[s]);
        }
        // ---- normalise, store
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            float l = l_run[h];
            l += __shfl_xor_sync(0xffffffffu, l, 1);
            l += __shfl_xor_sync(0xffffffffu, l, 2);
            const float inv = l > 0.f ? 1.f / l : 0.f;
            const int qrow = q0 + cw * 64 + wr * 16 + (lane >> 2) + 8 * h;
            if (qrow < a.sq) {
                __half* orow = a.o + static_cast<long long>(b) * a.o_bs + static_cast<long long>(qrow) * a.o_ss + head * HD;
#pragma unroll
                for (int jj = 0; jj < HD / 8; ++jj)
                    *reinterpret_cast<uint32_t*>(orow + 8 * jj + 2 * quad) =
                        pack_half2(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
            }
        }
    }
}

bool g_attr_set = false;

}  // namespace

bool attention_tc_eligible(const AttnParams& p) {
    if (p.head_dim != HD || p.b_inner != 1 || p.kv_batch_div < 1) return false;
    if (p.sq < 2 * BQ || p.skv < BKV) return false;                 // short sequences stay on the warp-MMA kernel
    const long long strides[] = {p.q_bs, p.q_ss, p.k_bs, p.k_ss, p.v_bs, p.v_ss};
    for (long long s : strides)
        if (s <= 0 || (s & 7) != 0) return false;                   // TMA: 16 B multiples
    if ((p.o_bs & 1) != 0 || (p.o_ss & 1) != 0) return false;       // fp16 pairs per store
    const uintptr_t ptrs[] = {reinterpret_cast<uintptr_t>(p.q), reinterpret_cast<uintptr_t>(p.k),
                              reinterpret_cast<uintptr_t>(p.v)};
    for (uintptr_t x : ptrs)
        if (x & 15) return false;
    if (reinterpret_cast<uintptr_t>(p.o) & 3) return false;
    if (p.heads > 65535 || p.batch > 65535) return false;
    return true;
}

int attention_tc(const AttnParams& p, cudaStream_t stream) {
    if (!attention_tc_eligible(p)) return -1;
    if (!g_attr_set) {
        if (cudaFuncSetAttribute(attention_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_TOTAL) != cudaSuccess) {
            fprintf(stderr, "[t2v] attention_tc: cudaFuncSetAttribute failed: %s\n", cudaGetErrorString(cudaGetLastError()));
            return -2;
        }
        g_attr_set = true;
    }
    CUtensorMap map_q, map_k, map_v;   // rank 3: (heads*64, sequence, batch)
    const unsigned box[3] = {HD, BQ, 1};
    const int kvb = (p.batch + p.kv_batch_div - 1) / p.kv_batch_div;
    struct {
        CUtensorMap* m;
        const __half* base;
        long long bs, ss;
        int S, nb;
    } maps[3] = {{&map_q, p.q, p.q_bs, p.q_ss, p.sq, p.batch},
                 {&map_k, p.k, p.k_bs, p.k_ss, p.skv, kvb},
                 {&map_v, p.v, p.v_bs, p.v_ss, p.skv, kvb}};
    for (auto& m : maps) {
        const unsigned long long dims[3] = {static_cast<unsigned long long>(p.heads) * HD, static_cast<unsigned long long>(m.S),
                                            static_cast<unsigned long long>(m.nb)};
        const unsigned long long str[2] = {static_cast<unsigned long long>(m.ss) * 2, static_cast<unsigned long long>(m.bs) * 2};
        if (tma_encode_f16(m.m, m.base, 3, dims, str, box) != 0) return -3;
    }
    Args a;
    a.o = p.o;
    a.o_bs = p.o_bs;
    a.o_ss = p.o_ss;
    a.sq = p.sq;
    a.skv = p.skv;
    a.kv_batch_div = p.kv_batch_div;
    a.n_kv = (p.skv + BKV - 1) / BKV;
    a.sl2 = p.scale * 1.4426950408889634f;
    dim3 grid((p.sq + BQ - 1) / BQ, p.heads, p.batch);
    attention_tc_kernel<<<grid, NTHREADS, SMEM_TOTAL, stream>>>(map_q, map_k, map_v, a);
    return launch_status("attention_tc launch");
}

}  // namespace t2v
