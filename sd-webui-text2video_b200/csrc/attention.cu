// softmax(Q K^T * scale) V with arbitrary (batch, sequence) strides, so that ONE kernel serves
//   * spatial self-attention   (batch = frame,    sequence = h*w tokens,  stride = row pitch)
//   * CLIP cross-attention     (batch = frame,    K/V = 77 text tokens shared by all frames of a sample)
//   * temporal self-attention  (batch = pixel,    sequence = frames,      stride = h*w * row pitch)
// directly on the channels-last token matrices -- the reference's (b h w) f c / b (h w) c rearranges
// (t2v_model.py:548-583, :727-761) never materialise.
//
// This file: flash-style online softmax with warp-level mma.sync.m16n8k16 (fp16 in, fp32 accumulate, fp32 softmax,
// P rounded to fp16 for P.V -- the numerics of torch SDPA's fused kernels that the reference dispatches to on the GPU,
// t2v_model.py:566-569).  One body serves every head width through two entry points:
//   * attention_kernel<TS>      head width 64: the SHORT sequences -- temporal attention (S = frames, 32 x 32 tiles),
//                               cross-attention (77 keys) and the coarse levels (h*w < 256).  Long spatial sequences go to
//                               the wgmma kernel in attention_tc.cu.
//   * attention_hd_kernel<HD>   head widths 8 / 16 / 32 / 40 / 80 / 160 (VideoCrafter: C/8 = 40 / 80 / 160), the spatial
//                               self-attention and CLIP cross-attention of CrossAttention.forward
//                               (videocrafter/lvdm/models/modules/attention_temporal.py:167-190), 64 x 64 tiles.
// attention() picks the route for every caller.

#include <type_traits>

#include "common.cuh"
#include "kernels.cuh"
#include "ptx.cuh"

namespace t2v {

namespace {

// Head width 64: 128 B rows, 16 B chunks XOR-swizzled by (row & 7) -> conflict-free ldmatrix
struct SwizzledTile {
    static constexpr int HDP = 64;
    static __device__ __forceinline__ uint32_t off(int row, int chunk) { return row * 128 + ((chunk ^ (row & 7)) << 4); }
    template <int TS>
    static __device__ __forceinline__ void load(uint32_t smem_tile, const __half* gbase, long long seq_stride, int s0,
                                                int s_len, int tid) {
        // TS rows x 8 chunks of 16 B, 2*TS threads -> 4 each
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int idx = tid + i * (2 * TS);
            const int row = idx >> 3;
            const int chunk = idx & 7;
            const bool ok = (s0 + row) < s_len;
            const __half* src = gbase + static_cast<long long>(ok ? (s0 + row) : 0) * seq_stride + chunk * 8;
            cp_async16(smem_tile + off(row, chunk), src, ok);
        }
    }
};

// The layout follows from the head width: the swizzle needs HD/8 to be a power of two, the padded pitch does not.
template <int HD>
using FlashTile = std::conditional_t<HD == 64, SwizzledTile, PaddedTile<HD>>;

// One CTA: TS queries of one (batch, head), 2*TS threads (16 query rows per warp), K/V streamed in TS-key tiles through
// two shared-memory stages sK[cur] / sV[cur].  The caller places the tiles.
template <int HD, int TS>
__device__ __forceinline__ void flash_attention(const AttnParams& p, uint32_t sQ, const uint32_t (&sK)[2],
                                                const uint32_t (&sV)[2]) {
    using Tile = FlashTile<HD>;
    constexpr int HDP = Tile::HDP;
    constexpr int NB = TS / 8, KSK = TS / 16;          // 8-key blocks of S, 16-key steps of P.V
    constexpr int KS = HDP / 16, NBD = HDP / 8;        // 16-dim steps of Q.K^T, 8-dim blocks of O
    const int tid = threadIdx.x;
    const int warp = tid >> 5;
    const int lane = tid & 31;
    const int q0 = blockIdx.z * TS;
    const int head = blockIdx.y;
    const int b = blockIdx.x;
    const int bkv = b / p.kv_batch_div;
    const long long bo = b / p.b_inner, bi = b % p.b_inner;
    const long long ko = bkv / p.b_inner, ki = bkv % p.b_inner;

    const __half* Q = p.q + bo * p.q_bs + bi * p.q_bsi + head * HD;
    const __half* K = p.k + ko * p.k_bs + ki * p.k_bsi + head * HD;
    const __half* V = p.v + ko * p.v_bs + ki * p.v_bsi + head * HD;
    __half* O = p.o + bo * p.o_bs + bi * p.o_bsi + head * HD;

    Tile::template load<TS>(sQ, Q, p.q_ss, q0, p.sq, tid);
    Tile::template load<TS>(sK[0], K, p.k_ss, 0, p.skv, tid);
    Tile::template load<TS>(sV[0], V, p.v_ss, 0, p.skv, tid);
    cp_async_commit();

    const int n_kv = (p.skv + TS - 1) / TS;
    const float sl2 = p.scale * 1.4426950408889634f;   // softmax scale folded into exp2

    uint32_t qf[KS][4];            // Q A-fragments for the k-steps over the head dim (16 dims each)
    float o_acc[NBD][4];           // 16 x HDP output tile: n-blocks of 8 dims
    float m_run[2] = {-INFINITY, -INFINITY};
    float l_run[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < NBD; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) o_acc[i][j] = 0.f;

    for (int it = 0; it < n_kv; ++it) {
        const int cur = it & 1;
        if (it + 1 < n_kv) {
            Tile::template load<TS>(sK[cur ^ 1], K, p.k_ss, (it + 1) * TS, p.skv, tid);
            Tile::template load<TS>(sV[cur ^ 1], V, p.v_ss, (it + 1) * TS, p.skv, tid);
            cp_async_commit();
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        if (it == 0) {
#pragma unroll
            for (int ks = 0; ks < KS; ++ks)
                ldmatrix_x4(qf[ks], sQ + Tile::off(warp * 16 + (lane & 15), ks * 2 + (lane >> 4)));
        }
        // ---- S = Q K^T (16 x TS per warp)
        float s[NB][4];
#pragma unroll
        for (int i = 0; i < NB; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) s[i][j] = 0.f;
#pragma unroll
        for (int ks = 0; ks < KS; ++ks) {
#pragma unroll
            for (int nb = 0; nb < NB; nb += 2) {
                uint32_t kf[4];
                // lanes 0-7: keys nb*8.., k-chunk 2ks ; 8-15: same keys, chunk 2ks+1 ; 16-31: next 8 keys
                const int row = nb * 8 + (lane & 7) + ((lane >> 4) << 3);
                const int chunk = ks * 2 + ((lane >> 3) & 1);
                ldmatrix_x4(kf, sK[cur] + Tile::off(row, chunk));
                const uint32_t b0[2] = {kf[0], kf[1]};
                const uint32_t b1[2] = {kf[2], kf[3]};
                mma_m16n8k16(s[nb], qf[ks], b0);
                mma_m16n8k16(s[nb + 1], qf[ks], b1);
            }
        }
        // ---- mask keys beyond skv, online softmax (rows g = lane/4 and g+8; cols 2*(lane%4)+{0,1} per n-block)
        const int kbase = it * TS;
        float m_new[2] = {m_run[0], m_run[1]};
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) {
            const int col = kbase + nb * 8 + (lane & 3) * 2;
            if (col >= p.skv) s[nb][0] = s[nb][2] = -INFINITY;
            if (col + 1 >= p.skv) s[nb][1] = s[nb][3] = -INFINITY;
            m_new[0] = fmaxf(m_new[0], fmaxf(s[nb][0], s[nb][1]));
            m_new[1] = fmaxf(m_new[1], fmaxf(s[nb][2], s[nb][3]));
        }
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            m_new[r] = fmaxf(m_new[r], __shfl_xor_sync(0xffffffffu, m_new[r], 1));
            m_new[r] = fmaxf(m_new[r], __shfl_xor_sync(0xffffffffu, m_new[r], 2));
        }
        float corr[2], msc[2];
#pragma unroll
        for (int r = 0; r < 2; ++r) {
            corr[r] = (m_run[r] == -INFINITY) ? 0.f : exp2f((m_run[r] - m_new[r]) * sl2);
            msc[r] = (m_new[r] == -INFINITY) ? 0.f : m_new[r] * sl2;
            m_run[r] = m_new[r];
            l_run[r] *= corr[r];
        }
        uint32_t pf[KSK][4];        // P as A-fragments for the key k-steps (16 keys each)
#pragma unroll
        for (int nb = 0; nb < NB; ++nb) {
            const float p0 = exp2f(s[nb][0] * sl2 - msc[0]);
            const float p1 = exp2f(s[nb][1] * sl2 - msc[0]);
            const float p2 = exp2f(s[nb][2] * sl2 - msc[1]);
            const float p3 = exp2f(s[nb][3] * sl2 - msc[1]);
            l_run[0] += p0 + p1;
            l_run[1] += p2 + p3;
            const __half2 h01 = __floats2half2_rn(p0, p1);
            const __half2 h23 = __floats2half2_rn(p2, p3);
            pf[nb >> 1][(nb & 1) * 2 + 0] = *reinterpret_cast<const uint32_t*>(&h01);
            pf[nb >> 1][(nb & 1) * 2 + 1] = *reinterpret_cast<const uint32_t*>(&h23);
        }
#pragma unroll
        for (int nb = 0; nb < NBD; ++nb) {
            o_acc[nb][0] *= corr[0];
            o_acc[nb][1] *= corr[0];
            o_acc[nb][2] *= corr[1];
            o_acc[nb][3] *= corr[1];
        }
        // ---- O += P V
#pragma unroll
        for (int ks = 0; ks < KSK; ++ks) {        // 16 keys per step
#pragma unroll
            for (int db = 0; db < NBD; db += 2) { // two 8-dim blocks per ldmatrix.x4.trans
                uint32_t vf[4];
                const int row = ks * 16 + (lane & 15);
                const int chunk = db + (lane >> 4);
                ldmatrix_x4_trans(vf, sV[cur] + Tile::off(row, chunk));
                const uint32_t b0[2] = {vf[0], vf[1]};
                const uint32_t b1[2] = {vf[2], vf[3]};
                mma_m16n8k16(o_acc[db], pf[ks], b0);
                mma_m16n8k16(o_acc[db + 1], pf[ks], b1);
            }
        }
        __syncthreads();   // everyone done with stage `cur` before it is refilled
    }
    // ---- finalize: divide by row sums, write fp16
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 1);
        l_run[r] += __shfl_xor_sync(0xffffffffu, l_run[r], 2);
    }
    const float inv[2] = {l_run[0] > 0.f ? 1.f / l_run[0] : 0.f, l_run[1] > 0.f ? 1.f / l_run[1] : 0.f};
    const int row0 = q0 + warp * 16 + (lane >> 2);
#pragma unroll
    for (int nb = 0; nb < NBD; ++nb) {
        const int col = nb * 8 + (lane & 3) * 2;
        if (HDP != HD && col >= HD) continue;         // zero-padded head-dim columns
        if (row0 < p.sq)
            *reinterpret_cast<__half2*>(O + static_cast<long long>(row0) * p.o_ss + col) =
                __floats2half2_rn(o_acc[nb][0] * inv[0], o_acc[nb][1] * inv[0]);
        if (row0 + 8 < p.sq)
            *reinterpret_cast<__half2*>(O + static_cast<long long>(row0 + 8) * p.o_ss + col) =
                __floats2half2_rn(o_acc[nb][2] * inv[1], o_acc[nb][3] * inv[1]);
    }
}

// Head width 64.  TS = 64 (64 queries x 64 keys per iteration, 4 warps) for long sequences; TS = 32 (2 warps) for the
// short temporal sequences (S = frames = 24 would waste 63 % of a 64 x 64 tile).
template <int TS>
__global__ void __launch_bounds__(2 * TS) attention_kernel(AttnParams p) {
    constexpr int TB = TS * 128;   // tile bytes
    // Q | K0 | V0 | K1 | V1: single-tile problems (temporal attention: S = frames <= 32, the gather is latency-bound) are launched with
    // the first three tiles only -> 12 KB instead of 20 KB per 64-thread CTA, 18 instead of 11 resident CTAs per SM
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t sQ = smem_u32(smem);
    const uint32_t sK[2] = {sQ + TB, sQ + 3 * TB};
    const uint32_t sV[2] = {sQ + 2 * TB, sQ + 4 * TB};
    flash_attention<64, TS>(p, sQ, sK, sV);
}

// Every other head width, 64 x 64 tiles: Q | K0 | K1 | V0 | V1
template <int HD>
__global__ void __launch_bounds__(128) attention_hd_kernel(AttnParams p) {
    constexpr int TB = 64 * PaddedTile<HD>::PB;
    extern __shared__ __align__(128) uint8_t smem[];
    const uint32_t sQ = smem_u32(smem);
    const uint32_t sK[2] = {sQ + TB, sQ + 2 * TB};
    const uint32_t sV[2] = {sQ + 3 * TB, sQ + 4 * TB};
    flash_attention<HD, 64>(p, sQ, sK, sV);
}

// Grid (batch, heads, query tiles), its limits and the shared memory of the warp-MMA route for head width HD
template <int HD>
int launch_flash(const AttnParams& p, cudaStream_t stream) {
    const int ts = HD == 64 && p.sq <= 32 && p.skv <= 32 ? 32 : 64;
    const dim3 grid(p.batch, p.heads, (p.sq + ts - 1) / ts);
    if (grid.z > 65535 || grid.y > 65535) return -3;
    if constexpr (HD == 64) {
        const int n_kv = (p.skv + ts - 1) / ts;
        const size_t smem = static_cast<size_t>(ts) * 128 * (n_kv > 1 ? 5 : 3);
        if (ts == 32) attention_kernel<32><<<grid, 64, smem, stream>>>(p);
        else attention_kernel<64><<<grid, 128, smem, stream>>>(p);
    } else {
        constexpr int smem = 5 * 64 * PaddedTile<HD>::PB;
        static bool attr = false;
        if (!attr) {
            if (cudaFuncSetAttribute(attention_hd_kernel<HD>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
                return -4;
            attr = true;
        }
        attention_hd_kernel<HD><<<grid, 128, smem, stream>>>(p);
    }
    return launch_status("attention launch");
}

bool attention_args_aligned(const AttnParams& p) {
    return attention_operands_aligned("attention", {p.q, p.k, p.v},
                                      {p.q_bs, p.q_bsi, p.q_ss, p.k_bs, p.k_bsi, p.k_ss, p.v_bs, p.v_bsi, p.v_ss}, p.o,
                                      {p.o_bs, p.o_bsi, p.o_ss});
}

}  // namespace

bool attention_operands_aligned(const char* who, std::initializer_list<const void*> loads,
                                std::initializer_list<long long> load_strides, const void* o,
                                std::initializer_list<long long> o_strides) {
    for (const void* x : loads)
        if (reinterpret_cast<uintptr_t>(x) & 15) {
            set_error("%s: Q, K, V and any relative-position tables must be 16-byte aligned", who);
            return false;
        }
    for (long long s : load_strides)
        if (s & 7) {
            set_error("%s: Q, K and V strides must be multiples of 8 elements", who);
            return false;
        }
    bool o_ok = !(reinterpret_cast<uintptr_t>(o) & 3);
    for (long long s : o_strides) o_ok = o_ok && !(s & 1);
    if (!o_ok) {
        set_error("%s: O must be 4-byte aligned with even strides", who);
        return false;
    }
    return true;
}

int attention(const AttnParams& p, cudaStream_t stream) {
    if (p.sq <= 0 || p.skv <= 0 || p.kv_batch_div <= 0 || p.b_inner <= 0) return -1;
    if (attention_tc_eligible(p)) return attention_tc(p, stream);
    if (!attention_args_aligned(p)) return -1;
    switch (p.head_dim) {
        case 8: return launch_flash<8>(p, stream);
        case 16: return launch_flash<16>(p, stream);
        case 32: return launch_flash<32>(p, stream);
        case 40: return launch_flash<40>(p, stream);
        case 64: return launch_flash<64>(p, stream);
        case 80: return launch_flash<80>(p, stream);
        case 160: return launch_flash<160>(p, stream);
        default: return -1;
    }
}

}  // namespace t2v
