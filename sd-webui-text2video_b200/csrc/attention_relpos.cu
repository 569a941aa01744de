// Temporal attention of the VideoCrafter denoiser (SURVEY.md 8 a19) with relative-position key/value tables:
// attention_relpos_kernel<HD, RT> is TemporalCrossAttention.forward (videocrafter/lvdm/models/modules/
// attention_temporal.py:107-144) with RelativePosition (:46-65), context = x, T <= 32 frames per sequence (16 query
// frames per pass; relative positions beyond +-L are clamped to the end rows of the tables):
//    sim[t,s] = scale * (q_t . k_s + q_t . Rk[clamp(s-t)+L])
//    out[t]   = sum_s attn[t,s] v_s + sum_s attn[t,s] Rv[clamp(s-t)+L]
// Both table terms run on the tensor cores as dense products against the WHOLE table (Q Rk^T is [T x (2L+1)], attn is
// skewed into [T x (2L+1)] for the Rv product); the diagonal gather / scatter between the two index spaces goes through
// shared memory.
//
// Warp-level mma.sync.m16n8k16 (fp16 in, fp32 accumulate), fp32 softmax, P rounded to fp16 for the value products.
// Shared-memory tiles are PaddedTile (ptx.cuh) for every head width.
#include <algorithm>
#include <cstdio>

#include "common.cuh"
#include "kernels.cuh"
#include "ptx.cuh"

namespace t2v {

namespace {

constexpr int RJ = 48;         // relative-position rows (2L+1 <= 48), multiple of 16
constexpr int RP_WARPS = 4;

template <int HD, int RT>      // RT = 16 or 32: frames per sequence, padded
struct RelSmem {
    using G = PaddedTile<HD>;
    static constexpr int kTable = RJ * G::PB;                       // one table, padded rows
    static constexpr int kQKV = RT * G::PB;                         // one RT-row operand tile
    static constexpr int kC2 = 16 * RJ * 4;                         // fp32 [16][48] Q.Rk^T of the current 16-row block
    static constexpr int kP2Pitch = RJ * 2 + 16;                    // 112 B
    static constexpr int kP2 = 16 * kP2Pitch;
    static constexpr int kWarp = 3 * kQKV + kC2 + kP2;
    static constexpr int kTotal = 2 * kTable + RP_WARPS * kWarp;
};

template <int HD, int RT>
__global__ void __launch_bounds__(RP_WARPS * 32) attention_relpos_kernel(RelposParams p) {
    using G = PaddedTile<HD>;
    using SM = RelSmem<HD, RT>;
    constexpr int NBK = RT / 8;        // 8-wide key blocks
    constexpr int KSK = RT / 16;       // 16-key steps of the P.V product
    extern __shared__ __align__(128) uint8_t smem_dyn[];
    const uint32_t sTk = smem_u32(smem_dyn);
    const uint32_t sTv = sTk + SM::kTable;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t wbase = sTv + SM::kTable + warp * SM::kWarp;
    const uint32_t sQ = wbase, sK = wbase + SM::kQKV, sV = wbase + 2 * SM::kQKV;
    const uint32_t sC2 = wbase + 3 * SM::kQKV;
    const uint32_t sP2 = sC2 + SM::kC2;
    float* c2 = reinterpret_cast<float*>(smem_dyn + (sC2 - sTk));
    uint8_t* p2 = smem_dyn + (sP2 - sTk);

    // tables: rows >= 2L+1 zero
    const int L = p.max_rel;
    const int nrel = 2 * L + 1;
    G::load_rows(sTk, p.table_k, HD, 0, nrel, RJ, tid, RP_WARPS * 32);
    G::load_rows(sTv, p.table_v, HD, 0, nrel, RJ, tid, RP_WARPS * 32);
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();

    const float scale = p.scale;
    const int g = lane >> 2, qd = lane & 3;
    const int rsel = (lane & 7) + ((lane >> 4) << 3);
    const long long items = static_cast<long long>(p.n_seq) * p.heads;
    for (long long item = static_cast<long long>(blockIdx.x) * RP_WARPS + warp; item < items;
         item += static_cast<long long>(gridDim.x) * RP_WARPS) {
        const long long seq = item / p.heads;
        const int head = static_cast<int>(item - seq * p.heads);
        const long long so = seq / p.seq_inner, si = seq % p.seq_inner;
        const long long base = so * p.bs_outer + si * p.bs_inner + head * HD;
        G::load_rows(sQ, p.q + base, p.ss, 0, p.T, RT, lane, 32);
        G::load_rows(sK, p.k + base, p.ss, 0, p.T, RT, lane, 32);
        G::load_rows(sV, p.v + base, p.ss, 0, p.T, RT, lane, 32);
        cp_async_commit();
        cp_async_wait<0>();
        __syncwarp();
        __half* O = p.o + so * p.o_bs_outer + si * p.o_bs_inner + head * HD;

#pragma unroll 1
        for (int mb = 0; mb < RT / 16; ++mb) {             // 16 query frames at a time
            if (mb * 16 >= p.T) break;
            // clear the skewed-probability tile of this block
            for (int i = lane; i < SM::kP2 / 16; i += 32) *reinterpret_cast<uint4*>(p2 + i * 16) = make_uint4(0u, 0u, 0u, 0u);
            uint32_t qf[G::KS][4];
#pragma unroll
            for (int ks = 0; ks < G::KS; ++ks)
                ldmatrix_x4(qf[ks], sQ + (mb * 16 + (lane & 15)) * G::PB + (ks * 2 + (lane >> 4)) * 16);
            // ---- S1 = Q K^T (16 x RT), S2 = Q Rk^T (16 x 48)
            float s1[NBK][4], s2[RJ / 8][4];
#pragma unroll
            for (int i = 0; i < NBK; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) s1[i][j] = 0.f;
#pragma unroll
            for (int i = 0; i < RJ / 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) s2[i][j] = 0.f;
#pragma unroll
            for (int ks = 0; ks < G::KS; ++ks) {
                const int chunk = ks * 2 + ((lane >> 3) & 1);
#pragma unroll
                for (int nb = 0; nb < NBK; nb += 2) {
                    uint32_t kf[4];
                    ldmatrix_x4(kf, sK + (nb * 8 + rsel) * G::PB + chunk * 16);
                    const uint32_t b0[2] = {kf[0], kf[1]};
                    const uint32_t b1[2] = {kf[2], kf[3]};
                    mma_m16n8k16(s1[nb], qf[ks], b0);
                    mma_m16n8k16(s1[nb + 1], qf[ks], b1);
                }
#pragma unroll
                for (int nb = 0; nb < RJ / 8; nb += 2) {
                    uint32_t kf[4];
                    ldmatrix_x4(kf, sTk + (nb * 8 + rsel) * G::PB + chunk * 16);
                    const uint32_t b0[2] = {kf[0], kf[1]};
                    const uint32_t b1[2] = {kf[2], kf[3]};
                    mma_m16n8k16(s2[nb], qf[ks], b0);
                    mma_m16n8k16(s2[nb + 1], qf[ks], b1);
                }
            }
            // scatter S2 to smem [16][48] fp32
#pragma unroll
            for (int nb = 0; nb < RJ / 8; ++nb) {
                const int j = nb * 8 + qd * 2;
                *reinterpret_cast<float2*>(c2 + g * RJ + j) = make_float2(s2[nb][0], s2[nb][1]);
                *reinterpret_cast<float2*>(c2 + (g + 8) * RJ + j) = make_float2(s2[nb][2], s2[nb][3]);
            }
            __syncwarp();
            // ---- sim = scale * (S1 + S2[t][clamp(s - t) + L]); softmax over s
            float pr[NBK][4];
            float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
            for (int nb = 0; nb < NBK; ++nb)
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const int tl = g + ((c >> 1) << 3);                 // row inside the block
                    const int s = nb * 8 + qd * 2 + (c & 1);
                    int dlt = s - (mb * 16 + tl);
                    dlt = dlt < -L ? -L : (dlt > L ? L : dlt);
                    float v = (s1[nb][c] + c2[tl * RJ + dlt + L]) * scale;
                    if (s >= p.T) v = -INFINITY;
                    pr[nb][c] = v;
                    mx[c >> 1] = fmaxf(mx[c >> 1], v);
                }
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
                mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
            }
            float sum[2] = {0.f, 0.f};
#pragma unroll
            for (int nb = 0; nb < NBK; ++nb)
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const float e = __expf(pr[nb][c] - mx[c >> 1]);
                    pr[nb][c] = e;
                    sum[c >> 1] += e;
                }
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 1);
                sum[r] += __shfl_xor_sync(0xffffffffu, sum[r], 2);
            }
            const float inv[2] = {1.f / sum[0], 1.f / sum[1]};
            // ---- P (fp16) as MMA A fragments; skew into relative-position space: P2[t][clamp(s-t)+L] += attn[t][s].
            //      |s-t| < L hits a unique cell; everything clamped to the two end rows of the table is summed per row.
            uint32_t pf[KSK][4];
            float lo[2] = {0.f, 0.f}, hi[2] = {0.f, 0.f};
#pragma unroll
            for (int nb = 0; nb < NBK; ++nb) {
                const __half2 h01 = __floats2half2_rn(pr[nb][0] * inv[0], pr[nb][1] * inv[0]);
                const __half2 h23 = __floats2half2_rn(pr[nb][2] * inv[1], pr[nb][3] * inv[1]);
                pf[nb >> 1][(nb & 1) * 2 + 0] = *reinterpret_cast<const uint32_t*>(&h01);
                pf[nb >> 1][(nb & 1) * 2 + 1] = *reinterpret_cast<const uint32_t*>(&h23);
                const __half hv[4] = {__low2half(h01), __high2half(h01), __low2half(h23), __high2half(h23)};
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    const int tl = g + ((c >> 1) << 3);
                    const int s = nb * 8 + qd * 2 + (c & 1);
                    const int dlt = s - (mb * 16 + tl);
                    if (s >= p.T) continue;
                    if (dlt <= -L) lo[c >> 1] += __half2float(hv[c]);
                    else if (dlt >= L) hi[c >> 1] += __half2float(hv[c]);
                    else *reinterpret_cast<__half*>(p2 + tl * SM::kP2Pitch + (dlt + L) * 2) = hv[c];
                }
            }
#pragma unroll
            for (int r = 0; r < 2; ++r) {
                lo[r] += __shfl_xor_sync(0xffffffffu, lo[r], 1);
                lo[r] += __shfl_xor_sync(0xffffffffu, lo[r], 2);
                hi[r] += __shfl_xor_sync(0xffffffffu, hi[r], 1);
                hi[r] += __shfl_xor_sync(0xffffffffu, hi[r], 2);
            }
            if (qd == 0) {
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int tl = g + r * 8;
                    *reinterpret_cast<__half*>(p2 + tl * SM::kP2Pitch + 0) = __float2half_rn(lo[r]);
                    *reinterpret_cast<__half*>(p2 + tl * SM::kP2Pitch + (2 * L) * 2) = __float2half_rn(hi[r]);
                }
            }
            __syncwarp();
            // ---- out = P V + P2 Rv
            float o_acc[G::NBD][4];
#pragma unroll
            for (int i = 0; i < G::NBD; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) o_acc[i][j] = 0.f;
#pragma unroll
            for (int ks = 0; ks < KSK; ++ks) {
#pragma unroll
                for (int db = 0; db < G::NBD; db += 2) {
                    uint32_t vf[4];
                    ldmatrix_x4_trans(vf, sV + (ks * 16 + (lane & 15)) * G::PB + (db + (lane >> 4)) * 16);
                    const uint32_t b0[2] = {vf[0], vf[1]};
                    const uint32_t b1[2] = {vf[2], vf[3]};
                    mma_m16n8k16(o_acc[db], pf[ks], b0);
                    mma_m16n8k16(o_acc[db + 1], pf[ks], b1);
                }
            }
#pragma unroll
            for (int ks = 0; ks < RJ / 16; ++ks) {
                uint32_t af[4];
                ldmatrix_x4(af, sP2 + (lane & 15) * SM::kP2Pitch + (ks * 2 + (lane >> 4)) * 16);
#pragma unroll
                for (int db = 0; db < G::NBD; db += 2) {
                    uint32_t vf[4];
                    ldmatrix_x4_trans(vf, sTv + (ks * 16 + (lane & 15)) * G::PB + (db + (lane >> 4)) * 16);
                    const uint32_t b0[2] = {vf[0], vf[1]};
                    const uint32_t b1[2] = {vf[2], vf[3]};
                    mma_m16n8k16(o_acc[db], af, b0);
                    mma_m16n8k16(o_acc[db + 1], af, b1);
                }
            }
            const int t0 = mb * 16 + g;
#pragma unroll
            for (int nb = 0; nb < G::NBD; ++nb) {
                const int col = nb * 8 + qd * 2;
                if (col >= HD) continue;
                if (t0 < p.T) *reinterpret_cast<__half2*>(O + static_cast<long long>(t0) * p.o_ss + col) = __floats2half2_rn(o_acc[nb][0], o_acc[nb][1]);
                if (t0 + 8 < p.T)
                    *reinterpret_cast<__half2*>(O + static_cast<long long>(t0 + 8) * p.o_ss + col) = __floats2half2_rn(o_acc[nb][2], o_acc[nb][3]);
            }
            __syncwarp();      // c2 / P2 are rewritten by the next block, the operand tiles by the next item
        }
    }
}

template <int HD, int RT>
int launch_relpos_rt(const RelposParams& p, cudaStream_t stream) {
    using SM = RelSmem<HD, RT>;
    static bool attr = false;
    if (!attr) {
        if (cudaFuncSetAttribute(attention_relpos_kernel<HD, RT>, cudaFuncAttributeMaxDynamicSharedMemorySize, SM::kTotal) != cudaSuccess)
            return -4;
        attr = true;
    }
    const long long items = static_cast<long long>(p.n_seq) * p.heads;
    const long long want = (items + RP_WARPS - 1) / RP_WARPS;
    const unsigned grid = static_cast<unsigned>(std::min<long long>(want, static_cast<long long>(num_sms()) * 2));
    attention_relpos_kernel<HD, RT><<<grid, RP_WARPS * 32, SM::kTotal, stream>>>(p);
    return launch_status("attention_relpos launch");
}
template <int HD>
int launch_relpos(const RelposParams& p, cudaStream_t stream) {
    return p.T <= 16 ? launch_relpos_rt<HD, 16>(p, stream) : launch_relpos_rt<HD, 32>(p, stream);
}

}  // namespace

int attention_relpos(const RelposParams& p, cudaStream_t stream) {
    if (p.T < 1 || p.T > 32 || p.max_rel < 1 || 2 * p.max_rel + 1 > RJ || p.n_seq <= 0 || p.heads <= 0 || p.seq_inner <= 0)
        return -1;
    if (!attention_operands_aligned("attention_relpos", {p.q, p.k, p.v, p.table_k, p.table_v}, {p.bs_outer, p.bs_inner, p.ss},
                                    p.o, {p.o_bs_outer, p.o_bs_inner, p.o_ss}))
        return -1;
    switch (p.head_dim) {
        case 8: return launch_relpos<8>(p, stream);
        case 16: return launch_relpos<16>(p, stream);
        case 32: return launch_relpos<32>(p, stream);
        case 40: return launch_relpos<40>(p, stream);
        case 64: return launch_relpos<64>(p, stream);
        case 80: return launch_relpos<80>(p, stream);
        case 160: return launch_relpos<160>(p, stream);
        default: return -1;
    }
}

}  // namespace t2v
