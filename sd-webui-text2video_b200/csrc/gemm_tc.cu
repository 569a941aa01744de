// wgmma / TMA implicit-GEMM kernel (sm_90a).  See gemm_tc.cuh for the data model.
//
// Per CTA (persistent, 384 threads = 3 warpgroups, 1 CTA/SM):
//   warpgroup 0     TMA producer : one elected thread issues, per k-iteration, one A box (128 rows x 64 K, tap-shifted
//                                  coordinates, OOB = zero padding) + one B box (BN x 64 K) into a SWIZZLE_128B smem ring;
//                                  warp 1 copies each tile's per-column epilogue operands (bias, or the LayerNorm fold's
//                                  colsum / bias32) into shared memory
//   warpgroups 1, 2 consumers    : each owns 64 rows of the 128-row tile; per ring stage 4 k-steps of wgmma m64 x BN x 16
//                                  (both operands from shared memory) into fp32 registers, then the epilogue (alpha, bias,
//                                  LayerNorm fold, residual, GEGLU) into a shared fp16 output tile that one thread hands
//                                  to TMA bulk stores (epilogue_tile), so the tile's writes drain to HBM while the next
//                                  tile's MMAs run.
// The producer runs ahead into the next tile while the consumers are in the epilogue.  What the epilogue needs besides the
// accumulators is fetched before they are ready: the row table and LayerNorm row statistics at tile start, the column
// operands by warp 1, the residual by a TMA load into the output tile issued as the tile's main loop starts.
// Outputs TMA cannot address (rows that are not 16-byte aligned), fp32 split-K partials (a 128 x 256 x 4 B tile does not fit
// beside the ring) and the B-stationary variant, whose resident weights leave no room for an output tile, store through
// per-warp staging slabs instead (epilogue_warp).
// CG = 2: a cluster of two CTAs owns two consecutive M-tiles of the same N-tile; each CTA fetches half of the B box and
// TMA-multicasts it into both CTAs, so B crosses L2 -> SM once per pair.
// Roofline: tensor-bound (2*M*N*K*taps flop per launch) whenever K*taps is large; see DESIGN.md.
#include "common.cuh"
#include "gemm_tc.cuh"
#include "kernels.cuh"
#include "ptx.cuh"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>

namespace t2v {

namespace {

constexpr int kThreads = 384;
constexpr int kRegsProducer = 40;                            // setmaxnreg budgets: 128 x 40 + 256 x 232 <= 64 K registers
constexpr int kRegsConsumer = 232;
constexpr int kABytes = GEMM_BLOCK_M * GEMM_BLOCK_K * 2;     // 16 KB
constexpr int kSmemPerBlock = 227 * 1024;
constexpr int kSmemBudget = 216 * 1024;                      // B-stationary: resident weights + A ring
constexpr int kMaxStages = 8;
// Slab-path staging, per consumer warp: 8 rows x 128 B (half of the warp's 16 rows at a time).  The slabs share the space of
// the TMA path's output tile (a launch uses one of the two).
constexpr int kEpiRowBytes = 128;
constexpr int kSlabBytes = 8 * 8 * kEpiRowBytes;
// Global row index of each consumer warp's 16 rows (32-bit: gemm_plan rejects problems of 2^31 rows or more).
constexpr int kRowTabBytes = 8 * 16 * 4;

// The output tile of the TMA path: 128 rows x OUTW fp16, as column chunks of [128 rows x OCW columns], each the smem image of
// one TMA box.  OCW = 32 columns (64 B rows, SWIZZLE_64B) divides every tile width of 32 or more, so no box reaches into the
// next tile's columns; BN = 16 tiles use 16-column boxes (32 B rows, SWIZZLE_32B).
__host__ __device__ constexpr int out_chunk_cols(int outw) { return outw >= 32 ? 32 : 16; }
__host__ __device__ constexpr int out_chunks(int outw) { return (outw + out_chunk_cols(outw) - 1) / out_chunk_cols(outw); }

// SLAB: the layout without an output tile (slab stores only), whose ring keeps the stage the tile would take at BN 224 / 256.
template <int BN, bool SLAB = false>
struct Cfg {
    static constexpr int kBBytes = BN * GEMM_BLOCK_K * 2;
    static constexpr int kStageBytes = kABytes + kBBytes;
    static constexpr int kColBytes = BN * 8;      // (colsum, bias32) fp32 pairs, or the fp16 bias
    static constexpr int kTailBytes = 1024 /*align slack*/ + 256 /*barriers*/ + kRowTabBytes + kColBytes;
    // output tile (sized for the plain variant, whose tile is the wider one) or the slabs, whichever is larger
    static constexpr int kOutBytes = SLAB ? kSlabBytes : std::max(kSlabBytes, out_chunks(BN) * GEMM_BLOCK_M * out_chunk_cols(BN) * 2);
    static constexpr int kStages = std::min(kMaxStages, (kSmemPerBlock - kTailBytes - kOutBytes) / kStageBytes);
    static constexpr int kSmemBytes = kStages * kStageBytes + kOutBytes + kTailBytes;
    static constexpr int kBsSmemBytes = kSmemBudget + kSlabBytes + kTailBytes;
    static_assert(kSmemBytes <= kSmemPerBlock, "shared memory per block");
};
static_assert(Cfg<256>::kStages == 3 && Cfg<224>::kStages == 3 && Cfg<192>::kStages == 4 && Cfg<160>::kStages == 5 &&
                  Cfg<128>::kStages == 6 && Cfg<64>::kStages == 8 && Cfg<16>::kStages == 8,
              "ring depths next to the output tile");
static_assert(Cfg<256, true>::kStages == 4 && Cfg<224, true>::kStages == 4, "ring depths without the output tile");

// erf-form GELU x * Phi(x) (F.gelu default, t2v_model.py:821).  Phi(x) = 1/2 erfc(-x / sqrt 2); for z = |x| / sqrt 2
// erfc(z) = t (a1 + t (a2 + t (a3 + t (a4 + t a5)))) exp(-z^2), t = 1 / (1 + p z) (Abramowitz-Stegun 7.1.26, |error| <=
// 1.5e-7 -- three orders below the fp16 rounding the reference applies to the result).  2 MUFU (rcp, ex2) + 13 FMA-pipe
// instructions instead of erff's ~32.
__device__ __forceinline__ float gelu_erf(float x) {
    const float z = fabsf(x) * 0.70710678118654752440f;
    float t;
    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));
    float p = fmaf(t, 0.5f * 1.061405429f, 0.5f * -1.453152027f);
    p = fmaf(p, t, 0.5f * 1.421413741f);
    p = fmaf(p, t, 0.5f * -0.284496736f);
    p = fmaf(p, t, 0.5f * 0.254829592f);
    const float q = p * t * ex2_approx(z * z * -1.4426950408889634f);      // 1/2 erfc(z)
    return x * (x < 0.f ? q : 1.0f - q);
}

// Byte offset of (row r, byte b of the row) in a staging slab of 8 rows x `segs` 16 B segments.  The segment index
// L = r * segs + b / 16 is XOR-swizzled with L / 8, so that the fragment side (8 rows, the same 16 B column of each) and the
// row side (8 consecutive segments per quarter-warp) both touch 8 distinct 16 B bank groups.
__device__ __forceinline__ uint32_t stg_off(int r, int b, int segs) {
    const int L = r * segs + (b >> 4);
    return static_cast<uint32_t>(((L ^ ((L >> 3) & 7)) << 4) | (b & 15));
}

// Step 1 of a warp's epilogue, in place on its accumulators (fragment layout, ptx.cuh): alpha + bias, or the LayerNorm fold
// (rs: (mean, rstd) of rows fr and fr + 8).  The tile's per-column operands come from `cols`, which the producer warpgroup
// filled (zero past N): (colsum, bias32) fp32 pairs with the fold, else the fp16 bias.  A per-sample bias (bias_rows > 0,
// where one tile's rows may fall into two samples) is read from global memory instead.
template <int BN, bool GEGLU>
__device__ __forceinline__ void epilogue_affine(const GemmDesc& g, float (&acc)[BN / 2], const uint8_t* cols, const int* rowg,
                                                const float2 (&rs)[2], int tn, int lane) {
    const int quad = lane & 3, fr = lane >> 2;           // fragment: rows fr, fr + 8; columns 8j + 2 quad + {0, 1}
    if (!GEGLU && g.bias != nullptr && g.bias_rows > 0 && (g.flags & GEMM_LN) == 0) {      // (gemm_plan: not with GEGLU)
        const int col0 = tn * BN + 2 * quad;                 // column of acc[0]
        const int nrem = g.N - col0;                         // acc[4j + e] is inside the problem while 8j + e < nrem
        const __half* brow[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int fg = rowg[fr + 8 * h];
            brow[h] = g.bias + (fg >= 0 ? (fg / g.bias_rows) * g.bias_stride : 0) + col0;
        }
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                if (8 * j + e >= nrem) continue;
                acc[4 * j + e] = fmaf(acc[4 * j + e], g.alpha, __half2float(__ldg(brow[0] + 8 * j + e)));
                acc[4 * j + 2 + e] = fmaf(acc[4 * j + 2 + e], g.alpha, __half2float(__ldg(brow[1] + 8 * j + e)));
            }
        }
        return;
    }
    const bool ln = (g.flags & GEMM_LN) != 0;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
        const int c = 8 * j + 2 * quad;                      // tile column of acc[4j], acc[4j + 2]; c + 1: acc[4j + 1], acc[4j + 3]
        if (ln) {
            const float4 p = *reinterpret_cast<const float4*>(cols + 8 * c);      // colsum, bias32 of c; colsum, bias32 of c + 1
            acc[4 * j] = fmaf(rs[0].y, fmaf(-rs[0].x, p.x, acc[4 * j]), p.y);
            acc[4 * j + 2] = fmaf(rs[1].y, fmaf(-rs[1].x, p.x, acc[4 * j + 2]), p.y);
            acc[4 * j + 1] = fmaf(rs[0].y, fmaf(-rs[0].x, p.z, acc[4 * j + 1]), p.w);
            acc[4 * j + 3] = fmaf(rs[1].y, fmaf(-rs[1].x, p.z, acc[4 * j + 3]), p.w);
        } else {
            const float2 b = __half22float2(*reinterpret_cast<const __half2*>(cols + 2 * c));
            acc[4 * j] = fmaf(acc[4 * j], g.alpha, b.x);
            acc[4 * j + 2] = fmaf(acc[4 * j + 2], g.alpha, b.x);
            acc[4 * j + 1] = fmaf(acc[4 * j + 1], g.alpha, b.y);
            acc[4 * j + 3] = fmaf(acc[4 * j + 3], g.alpha, b.y);
        }
    }
}

// Slab path: the residual of the fp16 epilogue, unit by unit (a unit = 128 B of output per row for 8 rows: chunk u / 2, rows 8 (u % 2) ..
// 8 (u % 2) + 7), in the row-side layout of the staging slab: 16 B per thread.  kResUnits units of a tile are in flight at
// a time; the first ones are issued while the tile's last MMAs run.  BN <= 192: the warp's whole slice (<= 12 x 16 B per
// thread); wider tiles keep four units in flight, which fits their register budget without spills.
template <int BN>
struct ResQ {
    static constexpr int kCW = kEpiRowBytes / 2;                       // output columns per unit
    static constexpr int kUnits = 2 * ((BN + kCW - 1) / kCW);
    static constexpr int kDepth = BN <= 192 ? kUnits : 4;
    static __device__ __forceinline__ int segs(int c) { return (min(kCW, BN - c * kCW) * 2) / 16; }
    static __device__ __forceinline__ void load(const GemmDesc& g, const int* rowg, int tn, int u, int lane, uint4 (&rb)[2]) {
        const int c = u >> 1, h = u & 1, sg = segs(c);
        const bool vec_res = (g.ldr & 7) == 0 && (reinterpret_cast<uintptr_t>(g.residual) & 15) == 0;
#pragma unroll
        for (int p = 0; p < 2; ++p) {
            const int idx = lane + 32 * p;
            rb[p] = make_uint4(0u, 0u, 0u, 0u);
            if (idx >= 8 * sg) continue;
            const int gr = rowg[8 * h + idx / sg];
            const int col = tn * BN + c * kCW + 8 * (idx % sg);
            if (gr < 0) continue;
            const __half* src = g.residual + gr * g.ldr + col;
            if (vec_res && col + 8 <= g.N) {
                rb[p] = __ldg(reinterpret_cast<const uint4*>(src));
            } else {
                uint32_t w[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                    const __half2 v = __halves2half2(col + 2 * e < g.N ? src[2 * e] : __ushort_as_half(0),
                                                     col + 2 * e + 1 < g.N ? src[2 * e + 1] : __ushort_as_half(0));
                    w[e] = *reinterpret_cast<const uint32_t*>(&v);
                }
                rb[p] = make_uint4(w[0], w[1], w[2], w[3]);
            }
        }
    }
};

// Step 2 of a warp's epilogue on the slab path: its 16 rows x BN accumulator columns -> global memory, per unit (chunk of
// 128 B of output per row, half h = rows 8h .. 8h + 7).  The residual slice (queued in rq, ResQ) goes into the staging slab;
// each thread adds it
// to its fragment values, rounds, and writes the result back to the same place; then the rows leave with 16 B stores.
// Per element the arithmetic is that of a direct store: fp32 affine, + residual in fp32, one rounding (GEGLU: fp16 value,
// fp16 gate, fp16 gelu, fp16 product).  fp32 output (split-K partials) stages 32 columns per unit and has no residual
// (gemm_plan), nor has GEGLU.  A segment that is cut by N, or an unaligned output / residual, goes element-wise.
// rowg[16]: global row of each of the warp's rows, -1 for rows outside the problem.
template <int BN, bool GEGLU, bool F32>
__device__ __forceinline__ void epilogue_warp(const GemmDesc& g, float (&acc)[BN / 2], uint4 (&rq)[ResQ<BN>::kDepth][2],
                                              uint8_t* stg, const int* rowg, int tn, int sp, int lane) {
    static_assert(!(GEGLU && F32), "GEGLU stores fp16");
    constexpr bool RES = !GEGLU && !F32;                 // the variants that may add a residual
    constexpr int ES = F32 ? 4 : 2;                      // output element bytes
    constexpr int EPS = 16 / ES;                         // elements per 16 B segment
    constexpr int OUTW = GEGLU ? BN / 2 : BN;            // output columns of the tile
    constexpr int CW = kEpiRowBytes / ES;                // output columns per unit
    constexpr int NCH = (OUTW + CW - 1) / CW;
    constexpr int NU = 2 * NCH;                          // units: (chunk u / 2, half u % 2)
    constexpr int QD = ResQ<BN>::kDepth;
    const int quad = lane & 3, fr = lane >> 2;           // fragment: rows fr, fr + 8; columns 8j + 2 quad + {0, 1}
    const int nvalid = GEGLU ? g.N / 2 : g.N;
    const int ocol0 = tn * OUTW;
    const bool has_res = RES && g.residual != nullptr;
    const bool vec_out = (g.ldo % EPS) == 0 && (reinterpret_cast<uintptr_t>(g.out) & 15) == 0 && (!F32 || (g.split_stride % EPS) == 0);

    auto segs_of = [](int c) { return (min(CW, OUTW - c * CW) * ES) / 16; };
#pragma unroll
    for (int u = 0; u < NU; ++u) {
        const int c = u >> 1, h = u & 1, segs = segs_of(c);
        if (RES && has_res) {
#pragma unroll
            for (int p = 0; p < 2; ++p) {
                const int idx = lane + 32 * p;
                if (idx < 8 * segs) *reinterpret_cast<uint4*>(stg + stg_off(idx / segs, 16 * (idx % segs), segs)) = rq[u % QD][p];
            }
            if (u + QD < NU) ResQ<BN>::load(g, rowg, tn, u + QD, lane, rq[u % QD]);
            __syncwarp();
        }
        // fragment side: row fr of this half, the chunk's columns
#pragma unroll
        for (int jj = 0; jj < CW / 8; ++jj) {
            if (jj >= segs * EPS / 8) break;
            const int j = c * (CW / 8) + jj;
            uint8_t* sp_ = stg + stg_off(fr, (8 * jj + 2 * quad) * ES, segs);
            float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
            if constexpr (GEGLU) {
                // out = fp16(value) * fp16(gelu(fp16(gate))): the reference's rounding points under autocast (t2v_model.py:819-821)
                const __half2 xh = __floats2half2_rn(v0, v1);
                const float2 gf = __half22float2(__floats2half2_rn(acc[BN / 4 + 4 * j + 2 * h], acc[BN / 4 + 4 * j + 2 * h + 1]));
                const __half2 ge = __floats2half2_rn(gelu_erf(gf.x), gelu_erf(gf.y));
                *reinterpret_cast<__half2*>(sp_) = __hmul2(xh, ge);          // fp16 x fp16 -> fp16 (RN)
            } else if constexpr (F32) {
                *reinterpret_cast<float2*>(sp_) = make_float2(v0, v1);
            } else {
                if (has_res) {
                    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(sp_));
                    v0 += f.x;
                    v1 += f.y;
                }
                *reinterpret_cast<__half2*>(sp_) = __floats2half2_rn(v0, v1);
            }
        }
        __syncwarp();
        // row side: 16 B per thread, whole row segments
#pragma unroll
        for (int p = 0; p < 2; ++p) {
            const int idx = lane + 32 * p;
            if (idx >= 8 * segs) continue;
            const int gr = rowg[8 * h + idx / segs];
            if (gr < 0) continue;
            const int col = ocol0 + c * CW + EPS * (idx % segs);
            const uint4 val = *reinterpret_cast<const uint4*>(stg + stg_off(idx / segs, 16 * (idx % segs), segs));
            uint8_t* dst = static_cast<uint8_t*>(g.out) + ((F32 ? sp * g.split_stride : 0) + gr * g.ldo + col) * ES;
            if (vec_out && col + EPS <= nvalid) {
                *reinterpret_cast<uint4*>(dst) = val;
            } else {
                const uint32_t w[4] = {val.x, val.y, val.z, val.w};
#pragma unroll
                for (int e = 0; e < EPS; ++e)
                    if (col + e < nvalid) {
                        if constexpr (F32) reinterpret_cast<uint32_t*>(dst)[e] = w[e];
                        else reinterpret_cast<uint16_t*>(dst)[e] = static_cast<uint16_t>(w[e >> 1] >> (16 * (e & 1)));
                    }
            }
        }
        __syncwarp();
    }
}

// Row-grid origin of M-tile tmi (the coordinates of its row 0 along d0 .. d_{nd-1}).
__device__ __forceinline__ void tile_origin(const GemmDesc& g, int tmi, int (&org)[GEMM_MAX_RDIMS]) {
#pragma unroll
    for (int d = 0; d < GEMM_MAX_RDIMS; ++d) org[d] = 0;
    if (g.nd == 1) {
        org[0] = tmi * g.box[0];
        return;
    }
    int tm = tmi;
#pragma unroll
    for (int d = 0; d < GEMM_MAX_RDIMS; ++d) {
        if (d < g.nd) {
            const int td = g.tdim[d];
            const int qd = tm / td;
            org[d] = (tm - qd * td) * g.box[d];
            tm = qd;
        }
    }
}

// One output-tile box (map_o / map_r: rank 1 + nd) at column c0 and row-grid origin org.
__device__ __forceinline__ void tma_store_box(const CUtensorMap* map, const void* src, int nd, int c0, const int (&org)[GEMM_MAX_RDIMS]) {
    if (nd == 1) tma_store_2d(map, src, c0, org[0]);
    else if (nd == 2) tma_store_3d(map, src, c0, org[0], org[1]);
    else if (nd == 3) tma_store_4d(map, src, c0, org[0], org[1], org[2]);
    else tma_store_5d(map, src, c0, org[0], org[1], org[2], org[3]);
}
__device__ __forceinline__ void tma_load_box(void* dst, const CUtensorMap* map, uint64_t* bar, int nd, int c0,
                                             const int (&org)[GEMM_MAX_RDIMS]) {
    if (nd == 1) tma_load_2d(dst, map, bar, c0, org[0]);
    else if (nd == 2) tma_load_3d(dst, map, bar, c0, org[0], org[1]);
    else if (nd == 3) tma_load_4d(dst, map, bar, c0, org[0], org[1], org[2]);
    else tma_load_5d(dst, map, bar, c0, org[0], org[1], org[2], org[3]);
}

// The output tile's chunks hold rows of OCW * 2 bytes whose 16 B units are XOR-swizzled as the TMA SWIZZLE_{64,32}B modes
// lay out a box: byte offset bits [4, 4 + log2(OCW / 8)) ^= bits [7, ...), which for a 1024 B aligned chunk are bits of the
// row index alone.  A warp's fragment writes (8 rows x 4 quads, one 16 B unit column) hit 32 distinct banks.
template <int OCW>
__device__ __forceinline__ int out_unit_swizzle(int r) { return ((r * OCW * 2) >> 7) & (OCW / 8 - 1); }

// Output chunks of tile column tn that hold columns < N (TMA path: the boxes stored, and loaded for the residual).
template <int BN, bool GEGLU>
__device__ __forceinline__ int live_out_chunks(const GemmDesc& g, int tn) {
    constexpr int OUTW = GEGLU ? BN / 2 : BN;
    constexpr int OCW = out_chunk_cols(OUTW);
    return min(out_chunks(OUTW), ((GEGLU ? g.N / 2 : g.N) - tn * OUTW + OCW - 1) / OCW);
}

// Step 2 of a warp's epilogue on the TMA path: the warp's 16 rows (r0 = its first tile row) go into the output tile, each
// value rounded once to fp16 after adding the residual that a TMA load put in the same place.  Per element the arithmetic is
// that of epilogue_warp.  The tile is free once tilefree completes (the store warp saw the previous tile's stores read it,
// and the residual landed); the warp then signals tilefull, and the store warp hands the tile to TMA stores.
template <int BN, bool GEGLU>
__device__ __forceinline__ void epilogue_tile(const GemmDesc& g, const float (&acc)[BN / 2], uint8_t* tile, uint64_t* tilefree,
                                              uint32_t tphase, uint64_t* tilefull, int r0, int lane) {
    constexpr int OUTW = GEGLU ? BN / 2 : BN;
    constexpr int OCW = out_chunk_cols(OUTW);
    const int quad = lane & 3, fr = lane >> 2;
    const bool has_res = !GEGLU && g.residual != nullptr;
    // rows r0 + fr and r0 + fr + 8 share the swizzle (it depends on row bits >= 1 below 8 only)
    const uint32_t row = smem_u32(tile) + static_cast<uint32_t>((r0 + fr) * (OCW * 2) + 4 * quad);      // shared address
    const int sw = out_unit_swizzle<OCW>(r0 + fr);
    mbar_wait(tilefree, tphase);
#pragma unroll
    for (int j = 0; j < OUTW / 8; ++j) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            // column 8j + 2 quad: chunk j / (OCW / 8), 16 B unit j % (OCW / 8) of the row
            const uint32_t p = row + (j / (OCW / 8)) * (GEMM_BLOCK_M * OCW * 2) + 8 * h * (OCW * 2) + (((j % (OCW / 8)) ^ sw) << 4);
            float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
            __half2 v;
            if constexpr (GEGLU) {
                // out = fp16(value) * fp16(gelu(fp16(gate))): the reference's rounding points under autocast (t2v_model.py:819-821)
                const __half2 xh = __floats2half2_rn(v0, v1);
                const float2 gf = __half22float2(__floats2half2_rn(acc[BN / 4 + 4 * j + 2 * h], acc[BN / 4 + 4 * j + 2 * h + 1]));
                v = __hmul2(xh, __floats2half2_rn(gelu_erf(gf.x), gelu_erf(gf.y)));
            } else {
                if (has_res) {
                    const uint32_t rw = ld_shared_u32(p);
                    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&rw));
                    v0 += f.x;
                    v1 += f.y;
                }
                v = __floats2half2_rn(v0, v1);
            }
            st_shared_u32(p, *reinterpret_cast<const uint32_t*>(&v));
        }
    }
    fence_proxy_async_smem();          // the writes are ordered before the TMA stores that read them
    __syncwarp();
    if (lane == 0) mbar_arrive(tilefull);
}

// BS = "B-stationary": the CTA keeps the WHOLE weight slice of its N-tile (all taps x K chunks) resident in shared memory and
// walks M-tiles of that N-tile only, so per tile just the A box moves through the ring.
template <int BN, bool GEGLU, int CG, bool BS = false, bool SLAB = false>
__global__ void __launch_bounds__(kThreads, 1) gemm_tc_kernel(const __grid_constant__ GemmDesc g) {
    using Cf = Cfg<BN, SLAB>;
    static_assert(!BS || CG == 1, "B-stationary tiles are single-CTA");
    static_assert(!BS || Cf::kBsSmemBytes <= kSmemPerBlock, "shared memory per block");
    constexpr int kBarStages = BS ? kMaxStages : Cf::kStages;      // barrier slots (BS: ring depth is a run-time value <= 8)
    const uint32_t rank = CG == 2 ? cluster_ctarank() : 0u;       // position in the cluster
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    uint8_t* smem = smem_raw + (((raw + 1023u) & ~1023u) - raw);   // SWIZZLE_128B atoms need 1024 B alignment
    // smem map: [ring][output tile | slabs][barriers][row table][column operands]
    // BS:       [resident B: k_total chunks of BN x 64][A ring: bs_stages x 16 KB] up to the fixed budget, then [slabs] ...
    uint8_t* const epi = smem + (BS ? kSmemBudget : Cf::kStages * Cf::kStageBytes);     // output tile (1024 B aligned) or slabs
    uint64_t* bars = reinterpret_cast<uint64_t*>(epi + (BS ? kSlabBytes : Cf::kOutBytes));
    uint64_t* full = bars;                       // [kStages] TMA -> consumers
    uint64_t* empty = bars + kBarStages;         // [kStages] consumers (of both CTAs of a cluster) -> TMA
    uint64_t* bfull = empty + kBarStages;        // BS: the resident weight slice has landed
    uint64_t* colfull = bfull + 1;               // column operands of the next tile are in `cols` (warp 1 -> consumers)
    uint64_t* colempty = bfull + 2;              // every consumer warp has read them (consumers -> warp 1)
    uint64_t* tilefree = bfull + 3;              // TMA path: the output tile may be written, residual in place (warp 2 -> consumers)
    uint64_t* tilefull = bfull + 4;              // every consumer warp has written its rows of the tile (consumers -> warp 2)
    int* const rowtab = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(bars) + 256);
    uint8_t* const cols = reinterpret_cast<uint8_t*>(rowtab) + kRowTabBytes;      // per-column epilogue operands, Cf::kColBytes
    const bool tma_out = !BS && !SLAB && g.tma_out != 0;         // else per-warp slabs (epilogue_warp)
    const int nst = BS ? g.bs_stages : Cf::kStages;
    uint8_t* const sB_res = smem;
    uint8_t* const sA_ring = smem + (BS ? g.ntaps * g.k_chunks * Cf::kBBytes : 0);

    const int wg = threadIdx.x >> 7;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&g.map_a);
        tma_prefetch_desc(&g.map_b);
        if (tma_out) {
            tma_prefetch_desc(&g.map_o);
            if (g.residual != nullptr) tma_prefetch_desc(&g.map_r);
        }
        for (int i = 0; i < kBarStages; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], 2 * CG);         // one arrival per consumer warpgroup of every CTA that writes this stage
        }
        if constexpr (BS) mbar_init(bfull, 1);
        mbar_init(colfull, 1);
        mbar_init(colempty, 8);                   // one arrival per consumer warp
        mbar_init(tilefree, 1);
        mbar_init(tilefull, 8);                   // one arrival per consumer warp
        fence_barrier_init();
    }
    if constexpr (CG == 2) cluster_sync_all();    // peer barriers are initialised before any multicast / remote arrive
    else __syncthreads();

    // work items: (pair of consecutive M-tiles, N-tile, K split); CTA `rank` of a cluster owns M-tile CG*pm + rank
    const int pairs_m = (g.tiles_m + CG - 1) / CG;
    const int nsplit = g.splits > 1 ? g.splits : 1;
    const int total_pairs = pairs_m * g.tiles_n * nsplit;
    const int k_total = g.ntaps * g.k_chunks;
    const int k_per = g.splits > 1 ? g.k_per_split : k_total;
    // BS: this CTA owns N-tile bs_tn and walks the M-tiles first_pair, first_pair + pair_stride, ... (work item = M-tile)
    const int bs_tn = BS ? static_cast<int>(blockIdx.x) % g.tiles_n : 0;
    const int first_pair = BS ? static_cast<int>(blockIdx.x) / g.tiles_n : static_cast<int>(blockIdx.x) / CG;
    const int pair_stride = BS ? (static_cast<int>(gridDim.x) - bs_tn + g.tiles_n - 1) / g.tiles_n : static_cast<int>(gridDim.x) / CG;
    const int total_items = BS ? g.tiles_m : total_pairs;
    // the per-column epilogue operands go through shared memory unless the bias is per sample (epilogue_affine)
    const bool col_operands = (g.flags & GEMM_LN) != 0 || g.bias == nullptr || g.bias_rows == 0;

    if (wg == 0) {
        // ------------------------------------------------------------------ TMA producer
        setmaxnreg_dec<kRegsProducer>();
        // One elected thread runs the whole loop (an elect.sync region compiles to single-threaded code for the uniform TMA
        // instructions).  Loop-invariant descriptor fields are hoisted into registers and (tap, K chunk) advance by counters.
        if (threadIdx.x < 32 && elect_one()) {
            int stage = 0;
            uint32_t phase = 0;
            if constexpr (BS) {
                if (first_pair < total_items) {        // the resident weight slice: every (tap, K chunk) box of N-tile bs_tn, once
                    mbar_expect_tx(bfull, static_cast<uint32_t>(k_total * Cf::kBBytes));
                    const int kch0 = g.k_chunks;
                    for (int it = 0, tap = 0, kc = 0; it < k_total; ++it) {
                        tma_load_3d(sB_res + it * Cf::kBBytes, &g.map_b, bfull, kc * GEMM_BLOCK_K, bs_tn * BN, tap);
                        if (++kc == kch0) {
                            kc = 0;
                            ++tap;
                        }
                    }
                }
            }
            const int kch = g.k_chunks, nd = g.nd, a_tx = g.a_tx_bytes, tiles_n_ = g.tiles_n, tiles_m_ = g.tiles_m;
            const int bdim = g.b_batch_dim;
            for (int wi = first_pair; wi < total_items; wi += pair_stride) {
                int sp = 0, pt = wi;
                if (!BS && nsplit > 1) {
                    sp = wi % nsplit;
                    pt = wi / nsplit;
                }
                const int it0 = sp * k_per, it1 = min(k_total, it0 + k_per);
                int tn = bs_tn, tmi = wi;
                if constexpr (!BS) {
                    const int pm = pt / tiles_n_;
                    tn = pt - pm * tiles_n_;
                    tmi = pm * CG + static_cast<int>(rank);
                }
                int org[GEMM_MAX_RDIMS];
                tile_origin(g, tmi, org);
                if (tmi >= tiles_m_) org[0] = g.dim[0];       // odd tail of a cluster: this CTA's tile is all out of bounds (zeros)
                const int bbatch = bdim < 0 ? 0 : (bdim == 0 ? org[0] : (bdim == 1 ? org[1] : (bdim == 2 ? org[2] : org[3])));
                int tap = 0, kc = it0;
                if (it0 >= kch) {
                    tap = it0 / kch;
                    kc = it0 - tap * kch;
                }
                int c1 = org[0] + g.tap_off[tap][0], c2 = org[1] + g.tap_off[tap][1];
                int c3 = org[2] + g.tap_off[tap][2], c4 = org[3] + g.tap_off[tap][3];
                for (int it = it0; it < it1; ++it) {
                    mbar_wait(&empty[stage], phase ^ 1u);
                    uint8_t* sa = BS ? sA_ring + stage * kABytes : smem + stage * Cf::kStageBytes;
                    uint8_t* sb = sa + kABytes;
                    const int k0 = kc * GEMM_BLOCK_K;
                    mbar_expect_tx(&full[stage], static_cast<uint32_t>(a_tx + (BS ? 0 : Cf::kBBytes)));
                    if (nd == 1) tma_load_2d(sa, &g.map_a, &full[stage], k0, c1);
                    else if (nd == 2) tma_load_3d(sa, &g.map_a, &full[stage], k0, c1, c2);
                    else if (nd == 3) tma_load_4d(sa, &g.map_a, &full[stage], k0, c1, c2, c3);
                    else tma_load_5d(sa, &g.map_a, &full[stage], k0, c1, c2, c3, c4);
                    if constexpr (CG == 2) {
                        // this CTA's half of the B box, into the same place of both CTAs' stage
                        constexpr int kHalf = BN / 2;
                        tma_load_3d_mc(sb + rank * (kHalf * GEMM_BLOCK_K * 2), &g.map_b, &full[stage], k0,
                                       tn * BN + static_cast<int>(rank) * kHalf, tap + bbatch, static_cast<uint16_t>(3));
                    } else if constexpr (!BS) {
                        tma_load_3d(sb, &g.map_b, &full[stage], k0, tn * BN, tap + bbatch);
                    }
                    if (++kc == kch) {              // next tap: new coordinate offsets (at most 9 times per tile)
                        kc = 0;
                        ++tap;
                        if (it + 1 < it1) {
                            c1 = org[0] + g.tap_off[tap][0];
                            c2 = org[1] + g.tap_off[tap][1];
                            c3 = org[2] + g.tap_off[tap][2];
                            c4 = org[3] + g.tap_off[tap][3];
                        }
                    }
                    if (++stage == nst) {
                        stage = 0;
                        phase ^= 1u;
                    }
                }
            }
        } else if (threadIdx.x >= 32 && threadIdx.x < 64 && col_operands) {
            // Warp 1: the per-column epilogue operands of each tile into `cols`, zero past N.  The consumers release the buffer
            // after step 1 of their epilogue, so the next tile's columns load during the rest of that epilogue and the next
            // main loop, off the consumers' path.
            const int lane = threadIdx.x & 31;
            const bool ln = (g.flags & GEMM_LN) != 0;
            uint32_t cphase = 0;
            for (int wi = first_pair; wi < total_items; wi += pair_stride) {
                const int col0 = (BS ? bs_tn : (wi / nsplit) % g.tiles_n) * BN;
                mbar_wait(colempty, cphase ^ 1u);
#pragma unroll
                for (int c = lane; c < BN; c += 32) {
                    const int col = col0 + c;
                    if (ln) {
                        reinterpret_cast<float2*>(cols)[c] =
                            col < g.N ? make_float2(__ldg(g.colsum + col), __ldg(g.bias32 + col)) : make_float2(0.f, 0.f);
                    } else {
                        reinterpret_cast<__half*>(cols)[c] = g.bias != nullptr && col < g.N ? __ldg(g.bias + col) : __ushort_as_half(0);
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(colfull);
                cphase ^= 1u;
            }
        } else if (threadIdx.x >= 64 && threadIdx.x < 96 && tma_out) {
            // Warp 2, TMA path: one thread moves each output tile.  It readies the tile for the consumers (residual boxes
            // loaded into it, or a plain arrival), waits until they have written it, hands it to TMA stores and waits only
            // until those have read the tile -- the writes drain to HBM while the consumers run the next tile's MMAs.  The
            // consumer warpgroups never wait on the stores themselves, which would hold back their warpgroup-wide wgmmas.
            if (elect_one()) {
                constexpr int OUTW = GEGLU ? BN / 2 : BN;
                constexpr int OCW = out_chunk_cols(OUTW);
                constexpr int kChunkBytes = GEMM_BLOCK_M * OCW * 2;
                const bool has_res = !GEGLU && g.residual != nullptr;
                const uint32_t box_bytes = static_cast<uint32_t>(g.a_tx_bytes / GEMM_BLOCK_K * OCW);    // box rows x OCW x 2 B
                uint32_t fphase = 0;
                for (int wi = first_pair; wi < total_items; wi += pair_stride) {
                    const int pt = wi / nsplit;
                    const int tn = pt % g.tiles_n;
                    const int tmi = (pt / g.tiles_n) * CG + static_cast<int>(rank);
                    const int nch = tmi < g.tiles_m ? live_out_chunks<BN, GEGLU>(g, tn) : 0;    // odd cluster tail: nothing
                    int org[GEMM_MAX_RDIMS];
                    tile_origin(g, tmi, org);
                    if (has_res && nch > 0) {
                        mbar_expect_tx(tilefree, nch * box_bytes);
                        for (int c = 0; c < nch; ++c)
                            tma_load_box(epi + c * kChunkBytes, &g.map_r, tilefree, g.nd, tn * OUTW + c * OCW, org);
                    } else {
                        mbar_arrive(tilefree);
                    }
                    mbar_wait(tilefull, fphase);
                    fphase ^= 1u;
                    for (int c = 0; c < nch; ++c) tma_store_box(&g.map_o, epi + c * kChunkBytes, g.nd, tn * OUTW + c * OCW, org);
                    bulk_commit_group();
                    bulk_wait_group_read_0();
                }
                bulk_wait_group_0();              // the shared memory outlives the stores
            }
        }
        __syncwarp();
    } else {
        // ------------------------------------------------------------------ consumers: MMA + epilogue
        setmaxnreg_inc<kRegsConsumer>();
        const int cw = wg - 1;                        // rows 64 cw .. 64 cw + 63 of the tile
        const int lt = threadIdx.x & 127;
        const int wr = lt >> 5, lane = lt & 31;
        int stage = 0;
        uint32_t phase = 0;
        if constexpr (BS) {
            if (first_pair < total_items) mbar_wait(bfull, 0u);
        }
        const bool out_f32 = (g.flags & GEMM_OUT_F32) != 0;
        const bool ln = (g.flags & GEMM_LN) != 0;
        uint8_t* const stg = epi + (cw * 4 + wr) * (8 * kEpiRowBytes);    // slab path: this warp's staging slab
        int* const rowg = rowtab + (cw * 4 + wr) * 16;                     // global row of each of the warp's 16 rows
        uint32_t cphase = 0, tphase = 0;
        float acc[BN / 2];
        uint4 rq[ResQ<BN>::kDepth][2];                                     // slab path: residual units in flight
        for (int wi = first_pair; wi < total_items; wi += pair_stride) {
            const int sp = BS ? 0 : wi % nsplit;
            const int pt = wi / nsplit;
            const int tn = BS ? bs_tn : pt % g.tiles_n;
            const int tmi = BS ? wi : (pt / g.tiles_n) * CG + static_cast<int>(rank);
            const int it0s = BS ? 0 : sp * k_per;
            const int k_iters = min(g.ntaps * g.k_chunks, it0s + k_per) - it0s;

            // ---- global row of each of this warp's 16 rows (-1: outside the problem) and the LayerNorm (mean, rstd) of the
            // thread's two fragment rows.  Both depend on the tile index only, so they are fetched before the main loop (the
            // previous tile's epilogue, which read the table, ended with __syncwarp).
            if (lane < 16) {
                const int r = cw * 64 + wr * 16 + lane;
                int grow = -1;
                if (tmi < g.tiles_m) {
                    if (g.nd == 1) {                       // plain row matrix: no div/mod chain
                        const int o = tmi * g.box[0];
                        if (r < g.box[0] && o + r < g.dim[0]) grow = o + r;
                    } else {
                        int tm = tmi, rr = r;
                        long long mul = 1, gr = 0;
                        bool valid = true;
#pragma unroll
                        for (int d = 0; d < GEMM_MAX_RDIMS; ++d) {
                            const int td = g.tdim[d];
                            const int c = (tm % td) * g.box[d] + rr % g.box[d];
                            tm /= td;
                            rr /= g.box[d];
                            valid = valid && (c < g.dim[d]);
                            gr += mul * c;
                            mul *= g.dim[d];
                        }
                        if (valid && rr == 0) grow = static_cast<int>(gr);
                    }
                }
                rowg[lane] = grow;
            }
            __syncwarp();
            float2 rs[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int fg = rowg[(lane >> 2) + 8 * h];
                rs[h] = ln && fg >= 0 ? __ldg(g.rowstat + fg) : make_float2(0.f, 1.f);
            }

            // ---- main loop: one ring stage per iteration, one wgmma group kept in flight
            int prev = -1;
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);       // the previous tile's epilogue reads stay before the MMAs
            for (int it = 0; it < k_iters; ++it) {
                mbar_wait(&full[stage], phase);
                const uint32_t sa = smem_u32(BS ? sA_ring + stage * kABytes : smem + stage * Cf::kStageBytes) + cw * (64 * 128);
                const uint32_t sb = BS ? smem_u32(sB_res + it * Cf::kBBytes) : smem_u32(smem + stage * Cf::kStageBytes) + kABytes;
                const uint64_t da = wgmma_desc_sw128(sa);
                const uint64_t db = wgmma_desc_sw128(sb);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < GEMM_BLOCK_K / 16; ++k)          // +32 B per K = 16 step (start address in 16 B units)
                    wgmma_ss<BN>(acc, da + static_cast<uint64_t>(k * 2), db + static_cast<uint64_t>(k * 2), (it | k) != 0 ? 1u : 0u);
                wgmma_commit();
                wgmma_wait<1>();                                      // the previous stage's group has retired
                if (prev >= 0 && lt == 0) {
                    mbar_arrive(&empty[prev]);
                    if constexpr (CG == 2) mbar_arrive_cluster(&empty[prev], rank ^ 1u);
                }
                prev = stage;
                if (++stage == nst) {
                    stage = 0;
                    phase ^= 1u;
                }
            }
            // slab path: the first residual units are in flight while the last MMAs run
            if constexpr (!GEGLU) {
                if (!tma_out && g.residual != nullptr) {
#pragma unroll
                    for (int u = 0; u < ResQ<BN>::kDepth; ++u) ResQ<BN>::load(g, rowg, tn, u, lane, rq[u]);
                }
            }
            wgmma_wait<0>();
#pragma unroll
            for (int i = 0; i < BN / 2; ++i) reg_fence(acc[i]);       // epilogue reads stay behind the wait
            if (prev >= 0 && lt == 0) {
                mbar_arrive(&empty[prev]);
                if constexpr (CG == 2) mbar_arrive_cluster(&empty[prev], rank ^ 1u);
            }

            // ---- epilogue: affine (column operands from `cols`, then the buffer goes back to warp 1), then the stores.  The
            // ring position crosses it packed into one opaque register (GEGLU, BN = 256 has none to spare).
            uint32_t ring = static_cast<uint32_t>(stage) | (phase << 16);
            asm volatile("" : "+r"(ring));
            if (col_operands) mbar_wait(colfull, cphase);
            epilogue_affine<BN, GEGLU>(g, acc, cols, rowg, rs, tn, lane);
            if (col_operands) {
                __syncwarp();
                if (lane == 0) mbar_arrive(colempty);
                cphase ^= 1u;
            }
            if (tma_out) {
                epilogue_tile<BN, GEGLU>(g, acc, epi, tilefree, tphase, tilefull, cw * 64 + wr * 16, lane);
                tphase ^= 1u;
            } else if constexpr (GEGLU) {
                epilogue_warp<BN, true, false>(g, acc, rq, stg, rowg, tn, sp, lane);
            } else if (out_f32) {
                epilogue_warp<BN, false, true>(g, acc, rq, stg, rowg, tn, sp, lane);
            } else {
                epilogue_warp<BN, false, false>(g, acc, rq, stg, rowg, tn, sp, lane);
            }
            asm volatile("" : "+r"(ring));
            stage = static_cast<int>(ring & 0xffffu);
            phase = ring >> 16;
        }
    }
    if constexpr (CG == 2) cluster_sync_all();    // no CTA may exit while its peer can still multicast into it or signal it
}

// ------------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode = nullptr;
bool g_inited = false;

int encode_map(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
               const cuuint32_t* box, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, static_cast<cuuint32_t>(rank), const_cast<void*>(base),
                          dims, strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        fprintf(stderr, "[t2v] cuTensorMapEncodeTiled failed: %d (rank %d, dims %llu %llu %llu %llu %llu)\n",
                static_cast<int>(r), rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
                (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0),
                (unsigned long long)(rank > 4 ? dims[4] : 0));
        return -1;
    }
    return 0;
}

// ---- (BN, GEGLU, CG) dispatch table
struct Variant {
    int bn, geglu, cg, smem;
    const void* fn;
    int bs, slab;
};
template <int BN, bool G, int CG>
Variant variant() {
    return Variant{BN, G ? 1 : 0, CG, Cfg<BN>::kSmemBytes, reinterpret_cast<const void*>(&gemm_tc_kernel<BN, G, CG>), 0, 0};
}
template <int BN, bool G>
Variant variant_bs() {
    return Variant{BN, G ? 1 : 0, 1, Cfg<BN>::kBsSmemBytes, reinterpret_cast<const void*>(&gemm_tc_kernel<BN, G, 1, true>), 1, 0};
}
template <int BN>
Variant variant_slab() {
    return Variant{BN, 0, 1, Cfg<BN, true>::kSmemBytes, reinterpret_cast<const void*>(&gemm_tc_kernel<BN, false, 1, false, true>), 0, 1};
}
const Variant* variants(int* n) {
    static const Variant v[] = {
        variant<16, false, 1>(),  variant<64, false, 1>(),  variant<128, false, 1>(), variant<160, false, 1>(),
        variant<192, false, 1>(), variant<224, false, 1>(),
        variant<256, false, 1>(), variant<64, true, 1>(),   variant<128, true, 1>(),  variant<256, true, 1>(),
        variant<64, false, 2>(),  variant<128, false, 2>(), variant<160, false, 2>(), variant<256, false, 2>(),
        variant<64, true, 2>(),   variant<128, true, 2>(),  variant<256, true, 2>(),
        variant_bs<160, false>(), variant_bs<128, false>(), variant_bs<128, true>(), variant_bs<64, false>(),
        variant_slab<224>(),      variant_slab<256>(),
    };
    *n = static_cast<int>(sizeof(v) / sizeof(v[0]));
    return v;
}
const Variant* find_variant(int bn, bool geglu, int cg, int bs, int slab) {
    int n;
    const Variant* v = variants(&n);
    for (int i = 0; i < n; ++i)
        if (v[i].bn == bn && v[i].geglu == (geglu ? 1 : 0) && v[i].cg == cg && v[i].bs == bs && v[i].slab == slab) return &v[i];
    return nullptr;
}

}  // namespace

int gemm_init() {
    if (g_inited) return 0;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) != cudaSuccess ||
        fn == nullptr) {
        fprintf(stderr, "[t2v] cuTensorMapEncodeTiled entry point not found\n");
        return -1;
    }
    g_encode = reinterpret_cast<EncodeTiledFn>(fn);
    int nv = 0;
    const Variant* vs = variants(&nv);
    bool attr_fail = false;
    for (int i = 0; i < nv; ++i)
        if (cudaFuncSetAttribute(vs[i].fn, cudaFuncAttributeMaxDynamicSharedMemorySize, vs[i].smem) != cudaSuccess) attr_fail = true;
    if (attr_fail) {
        fprintf(stderr, "[t2v] cudaFuncSetAttribute(max dynamic smem) failed: %s\n",
                cudaGetErrorString(cudaGetLastError()));
        return -1;
    }
    g_inited = true;
    return 0;
}

int tma_encode_f16(CUtensorMap* m, const void* base, int rank, const unsigned long long* dims,
                   const unsigned long long* strides_bytes, const unsigned* box) {
    if (gemm_init() != 0) return -1;
    cuuint64_t d[5], st[5];
    cuuint32_t bx[5];
    for (int i = 0; i < rank; ++i) {
        d[i] = dims[i];
        bx[i] = box[i];
        if (i + 1 < rank) st[i] = strides_bytes[i];
    }
    return encode_map(m, base, rank, d, st, bx);
}

// Tile width of the B-stationary variant for this problem (0 = not eligible).  tiles_m = ceil(rows / 128) for plain row
// matrices; any_k lifts the K limit.
static int gemm_bs_bn(long long tiles_m, int N, int K, int ntaps, int num_sms, int force_bn, bool any_k, int* stages_out) {
    static const bool bs_off = getenv("T2V_NO_BSTAT") != nullptr;
    // Off by default (not measured faster on the model's layers); opt-in with T2V_BSTAT_KMAX=<max K chunks>, e.g. 5, and taken
    // by the op-level tests (GEMM_DBG_FORCE_BS).
    static const int bs_kmax = getenv("T2V_BSTAT_KMAX") ? atoi(getenv("T2V_BSTAT_KMAX")) : 0;
    const int kt = ntaps * ((K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K);
    if (bs_off || N <= 16 || (kt > bs_kmax && !any_k)) return 0;
    const int cands[3] = {160, 128, 64};
    for (int i = 0; i < 3; ++i) {
        const int c = cands[i];
        if (force_bn != 0 && force_bn != c) continue;
        const int tn = (N + c - 1) / c;
        if (static_cast<double>(N) / (static_cast<double>(tn) * c) < 0.9) continue;
        const long long b_bytes = static_cast<long long>(kt) * c * GEMM_BLOCK_K * 2;
        if (b_bytes > kSmemBudget - 4 * kABytes || tn > num_sms) continue;
        const int stages = static_cast<int>(std::min<long long>(8, (kSmemBudget - b_bytes) / kABytes));
        const int group = num_sms / tn;                               // CTAs per N-tile
        if (tiles_m < 3LL * group) continue;                          // too few M-tiles per CTA to amortise the resident load
        if (stages_out) *stages_out = stages;
        return c;
    }
    return 0;
}

int gemm_plan(const GemmProblem& p, GemmPlan* plan, int num_sms) {
    if (gemm_init() != 0) return -1;
    if (p.nd < 1 || p.nd > GEMM_MAX_RDIMS || p.ntaps < 1 || p.ntaps > GEMM_MAX_TAPS) return -2;
    if ((p.lda & 7) != 0 || (p.K & 7) != 0 || (reinterpret_cast<uintptr_t>(p.a) & 15) != 0 ||
        (reinterpret_cast<uintptr_t>(p.b) & 15) != 0) {
        fprintf(stderr, "[t2v] gemm_plan: operands must be 16-byte aligned (lda %lld K %d)\n", p.lda, p.K);
        return -3;
    }
    GemmDesc& g = plan->desc;
    memset(&g, 0, sizeof(g));
    g.nd = p.nd;
    long long rows = 1;
    // ---- M tiling: fill a 128-row box from the fastest row dim outwards
    int remaining = GEMM_BLOCK_M;
    int boxrows = 1;
    for (int d = 0; d < GEMM_MAX_RDIMS; ++d) {
        const int ext = d < p.nd ? p.dim[d] : 1;
        g.dim[d] = ext;
        int b = std::min(ext, remaining);
        if (b < 1) b = 1;
        // keep boxes that do not cover a full dim a divisor-friendly size (avoid ragged interior tiles)
        g.box[d] = b;
        g.tdim[d] = (ext + b - 1) / b;
        remaining = b >= ext ? remaining / b : 1;     // only grow into the next dim when this one is fully covered
        boxrows *= b;
        rows *= ext;
    }
    if (rows >= (1LL << 31)) {          // the epilogue's row table holds 32-bit row indices
        fprintf(stderr, "[t2v] gemm_plan: %lld rows, at most 2^31 - 1\n", rows);
        return -4;
    }
    if (p.b_batch_dim >= 0 && g.box[p.b_batch_dim] != 1) {
        // a tile may not straddle two B batches: shrink that dim's box to 1
        const int d = p.b_batch_dim;
        boxrows /= g.box[d];
        g.box[d] = 1;
        g.tdim[d] = g.dim[d];
        for (int e = d + 1; e < GEMM_MAX_RDIMS; ++e) {   // outer dims were grown assuming d was covered
            boxrows /= g.box[e];
            g.box[e] = 1;
            g.tdim[e] = g.dim[e];
        }
    }
    g.tiles_m = 1;
    for (int d = 0; d < GEMM_MAX_RDIMS; ++d) g.tiles_m *= g.tdim[d];
    g.a_tx_bytes = boxrows * GEMM_BLOCK_K * 2;
    g.ntaps = p.ntaps;
    g.k_chunks = (p.K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K;
    for (int t = 0; t < p.ntaps; ++t)
        for (int d = 0; d < GEMM_MAX_RDIMS; ++d) g.tap_off[t][d] = static_cast<int8_t>(d < p.nd ? p.tap_off[t][d] : 0);
    g.b_batch_dim = p.b_batch_dim;
    g.N = p.N;
    g.flags = p.flags;
    g.out = p.out;
    g.ldo = p.ldo;
    g.bias = p.bias;
    g.bias_rows = p.bias_rows;
    g.bias_stride = p.bias_stride;
    g.residual = p.residual;
    g.ldr = p.ldr;
    g.alpha = p.alpha == 0.f ? 1.0f : p.alpha;
    g.rowstat = p.rowstat;
    g.colsum = p.colsum;
    g.bias32 = p.bias32;
    g.splits = gemm_split_count(p, p.splits);
    g.k_per_split = (g.ntaps * g.k_chunks + g.splits - 1) / g.splits;
    g.split_stride = p.split_stride;

    // ---- N tiling: the tile width with the shortest modelled kernel time.  A persistent CTA walks ceil(tiles / CTAs) tiles
    // whose main loop (K steps) and epilogue add up, plus the fill of the last wave.  So: as few K steps per CTA as possible --
    // wide tiles, even slightly padded ones (N = 1920 -> 9 x 224 instead of 12 x 160), unless the epilogue is the longer leg.
    int bn = p.force_bn;
    const int k_total_sel = p.ntaps * g.k_chunks;
    if (bn == 0 && k_total_sel >= 10) {
        // K-heavy tiles (>= 10 K steps): the MMA leg dominates -> time model, padded wide tiles allowed.
        const int cands[7] = {256, 224, 192, 160, 128, 64, 16};
        double best = 1e30;
        for (int i = 0; i < 7; ++i) {
            const int c = cands[i];
            if ((p.flags & GEMM_GEGLU) && c != 256 && c != 128 && c != 64) continue;
            if (c == 16 && p.N > 16) continue;
            if (c > 16 && p.N <= 16) continue;
            if ((c == 224 || c == 192) && ((p.flags & GEMM_GEGLU) || p.b_batch_dim >= 0 || p.splits > 1)) continue;   // plain variants only
            const int tn = (p.N + c - 1) / c;
            if ((p.flags & GEMM_GEGLU) && (p.N % c) != 0) continue;
            const long long tiles = static_cast<long long>(tn) * g.tiles_m * g.splits;
            const long long ctas = std::min<long long>(tiles, num_sms);
            const long long per_cta = (tiles + ctas - 1) / ctas;
            const int k_iters = g.splits > 1 ? (k_total_sel + g.splits - 1) / g.splits : k_total_sel;
            const double t_iter = std::max(650.0, 2.7 * c);
            const int chunks_per_warp = c >= 64 ? (c / 32 + 1) / 2 : 1;
            const double t_epi = 900.0 + chunks_per_warp * (p.residual != nullptr ? 2100.0 : 1050.0);
            const double t_tile = std::max(k_iters * t_iter, t_epi) + 1500.0;
            const double fit = static_cast<double>(p.N) / (static_cast<double>(tn) * c);
            const double t = (per_cta * t_tile + t_epi) * (1.0 + 0.02 * (1.0 - fit));
            if (t < best) {
                best = t;
                bn = c;
            }
        }
    }
    if (bn == 0) {
        // few K steps per tile (K = 320 layers): prologue / epilogue legs dominate and the measured optimum is the exact-fit width
        const int cands[5] = {256, 160, 128, 64, 16};
        const double eff[5] = {1.0, 0.86, 0.80, 0.55, 0.25};
        double best = -1;
        for (int i = 0; i < 5; ++i) {
            const int c = cands[i];
            if ((p.flags & GEMM_GEGLU) && c != 256 && c != 128 && c != 64) continue;
            if (c == 16 && p.N > 16) continue;
            if (c > 16 && p.N <= 16) continue;
            const int tn = (p.N + c - 1) / c;
            const double waste = static_cast<double>(p.N) / (static_cast<double>(tn) * c);
            const long long tiles = static_cast<long long>(tn) * g.tiles_m;
            const long long waves = (tiles + num_sms - 1) / num_sms;
            const double fill = static_cast<double>(tiles) / (static_cast<double>(waves) * num_sms);
            const double score = eff[i] * waste * fill;
            if (score > best) {
                best = score;
                bn = c;
            }
        }
    }
    // ---- B-stationary variant (see the kernel): few K chunks, many M-tiles per CTA.  Never for GEGLU: its epilogue gains
    // nothing from resident weights and loses with the 128-wide tiles they would need.
    plan->bs = 0;
    if (!(p.flags & GEMM_GEGLU) && p.force_bs >= 0 && p.force_cg <= 1 && p.splits <= 1 && p.b_batch_dim < 0) {
        int stages = 0;
        const int c = gemm_bs_bn(g.tiles_m, p.N, p.K, p.ntaps, num_sms, p.force_bn, p.force_bs == 1, &stages);
        if (c > 0) {
            bn = c;
            plan->bs = 1;
            g.bs_stages = stages;
        }
    }
    plan->bn = bn;
    // Clusters of two CTAs (two M-tiles, B halves multicast into both): opt-in (T2V_2CTA=1 or force_cg), not measured faster.
    static const bool use_pairs = getenv("T2V_2CTA") != nullptr;
    plan->cg = p.force_cg ? p.force_cg : ((g.tiles_m >= 2 && bn >= 64 && use_pairs) ? 2 : 1);
    if (bn < 64 || p.b_batch_dim >= 0 || plan->bs || bn == 192 || bn == 224) plan->cg = 1;     // a cluster shares ONE B tile: never across B batches
    g.tiles_n = (p.N + bn - 1) / bn;
    if ((p.flags & GEMM_OUT_F32) && p.residual != nullptr) {
        fprintf(stderr, "[t2v] gemm_plan: fp32 output takes no residual\n");
        return -4;
    }
    if ((p.flags & GEMM_GEGLU) && (p.N % bn) != 0) {
        fprintf(stderr, "[t2v] gemm_plan: GEGLU needs N %% BN == 0 (N %d BN %d)\n", p.N, bn);
        return -4;
    }
    if ((p.flags & GEMM_GEGLU) && ((p.ldo & 15) != 0 || (reinterpret_cast<uintptr_t>(p.out) & 31) != 0 || p.residual != nullptr ||
                                   (p.flags & GEMM_OUT_F32) || p.bias_rows != 0 || p.splits > 1)) {
        fprintf(stderr, "[t2v] gemm_plan: GEGLU epilogue needs 32-byte aligned fp16 output rows (ldo %lld), no residual, "
                        "no per-sample bias, no split-K\n", p.ldo);
        return -4;
    }

    // ---- tensor maps
    {
        cuuint64_t dims[5], strides[4];
        cuuint32_t box[5];
        dims[0] = static_cast<cuuint64_t>(p.K);
        box[0] = GEMM_BLOCK_K;
        long long pitch = p.lda * 2;       // bytes between consecutive rows
        for (int d = 0; d < p.nd; ++d) {
            dims[d + 1] = static_cast<cuuint64_t>(g.dim[d]);
            box[d + 1] = static_cast<cuuint32_t>(g.box[d]);
            strides[d] = static_cast<cuuint64_t>(pitch);
            pitch *= g.dim[d];
        }
        if (encode_map(&g.map_a, p.a, p.nd + 1, dims, strides, box) != 0) return -5;
    }
    {
        const int nb = p.b_batch_dim >= 0 ? g.dim[p.b_batch_dim] : p.ntaps;
        cuuint64_t dims[3] = {static_cast<cuuint64_t>(p.K), static_cast<cuuint64_t>(p.n_alloc),
                              static_cast<cuuint64_t>(nb)};
        const cuuint64_t ldb = static_cast<cuuint64_t>(p.ldb > 0 ? p.ldb : p.K);
        cuuint64_t strides[2] = {ldb * 2, ldb * 2 * static_cast<cuuint64_t>(p.n_alloc)};
        cuuint32_t box[3] = {GEMM_BLOCK_K, static_cast<cuuint32_t>(bn / plan->cg), 1};   // a CTA of a cluster fetches half of B
        if (encode_map(&g.map_b, p.b, 3, dims, strides, box) != 0) return -6;
    }
    // ---- output path: TMA stores from a shared output tile wherever TMA can address the fp16 output (and residual) rows;
    // per-warp slabs for fp32 output, rows that are not 16-byte aligned, and the B-stationary variant (no room for the tile)
    const auto tma_rows = [](const void* ptr, long long ld) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && (ld & 7) == 0; };
    g.tma_out = !(p.flags & GEMM_OUT_F32) && !plan->bs && !p.slab_out && tma_rows(p.out, p.ldo) &&
                (p.residual == nullptr || tma_rows(p.residual, p.ldr));
    // The stores of a tile drain behind the CTA's next tile; with no next tile (one wave: every CTA has at most one) or no
    // TMA stores at all (fp32 split-K partials, unaligned rows) the output tile only costs the 224 / 256-wide rings a stage,
    // so those launches take the variant without it (4 stages instead of 3; the K-heavy one-wave level-2 layers).
    const long long tiles_all = static_cast<long long>(g.tiles_m) * g.tiles_n * g.splits;
    plan->slab = !plan->bs && plan->cg == 1 && !(p.flags & GEMM_GEGLU) && (bn == 224 || bn == 256) &&
                 (!g.tma_out || tiles_all <= num_sms) ? 1 : 0;
    if (plan->slab) g.tma_out = 0;
    if (g.tma_out) {
        // rank 1 + nd over the same row grid as map_a: (output columns, d0, .., d_{nd-1}); box = one output-tile chunk
        const int outw = (p.flags & GEMM_GEGLU) ? bn / 2 : bn;
        const int ocw = out_chunk_cols(outw);
        cuuint64_t dims[5];
        cuuint64_t strides[4];
        cuuint32_t box[5];
        dims[0] = static_cast<cuuint64_t>((p.flags & GEMM_GEGLU) ? p.N / 2 : p.N);
        box[0] = static_cast<cuuint32_t>(ocw);
        for (int d = 0; d < p.nd; ++d) {
            dims[d + 1] = static_cast<cuuint64_t>(g.dim[d]);
            box[d + 1] = static_cast<cuuint32_t>(g.box[d]);
        }
        const CUtensorMapSwizzle sw = ocw == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B;
        for (int which = 0; which < (p.residual != nullptr ? 2 : 1); ++which) {
            long long pitch = (which == 0 ? p.ldo : p.ldr) * 2;
            for (int d = 0; d < p.nd; ++d) {
                strides[d] = static_cast<cuuint64_t>(pitch);
                pitch *= g.dim[d];
            }
            if (encode_map(which == 0 ? &g.map_o : &g.map_r, which == 0 ? p.out : p.residual, p.nd + 1, dims, strides, box, sw) != 0)
                return -8;
        }
    }
    const Variant* var = find_variant(bn, (p.flags & GEMM_GEGLU) != 0, plan->cg, plan->bs, plan->slab);
    if (var == nullptr) return -7;
    const long long pairs = static_cast<long long>((g.tiles_m + plan->cg - 1) / plan->cg) * g.tiles_n * g.splits;
    plan->grid = plan->cg * static_cast<int>(std::min<long long>(pairs, num_sms / plan->cg));
    if (plan->bs) plan->grid = (num_sms / g.tiles_n) * g.tiles_n;             // equal groups of CTAs per N-tile
    plan->smem = var->smem;
    plan->flops = 2.0 * static_cast<double>(rows) * p.N * p.K * p.ntaps;
    return 0;
}

int gemm_launch(const GemmPlan& plan, cudaStream_t stream) {
    const Variant* var = find_variant(plan.bn, (plan.desc.flags & GEMM_GEGLU) != 0, plan.cg, plan.bs, plan.slab);
    if (var == nullptr) return -1;
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = dim3(static_cast<unsigned>(plan.grid));
    cfg.blockDim = dim3(static_cast<unsigned>(kThreads));
    cfg.dynamicSmemBytes = static_cast<size_t>(plan.smem);
    cfg.stream = stream;
    cudaLaunchAttribute attr;
    attr.id = cudaLaunchAttributeClusterDimension;
    attr.val.clusterDim.x = 2;
    attr.val.clusterDim.y = 1;
    attr.val.clusterDim.z = 1;
    cfg.attrs = &attr;
    cfg.numAttrs = plan.cg == 2 ? 1 : 0;
    void* args[1] = {const_cast<GemmDesc*>(&plan.desc)};
    return cudaLaunchKernelExC(&cfg, var->fn, args) == cudaSuccess ? 0 : -2;
}

// ------------------------------------------------------------------------------------------ split-K
static long long problem_rows(const GemmProblem& p) {
    long long rows = 1;
    for (int d = 0; d < p.nd; ++d) rows *= p.dim[d];
    return rows;
}

int gemm_split_count(const GemmProblem& p, int requested) {
    if (requested <= 1) return 1;
    const int kt = p.ntaps * ((p.K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K);
    const int kps = (kt + requested - 1) / requested;
    return (kt + kps - 1) / kps;
}

const char* gemm_splitk_unsupported(const GemmProblem& p) {
    const auto a16 = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; };
    if (p.flags & GEMM_GEGLU) return "GEGLU epilogue";
    if (p.flags & GEMM_LN) return "LayerNorm-folded epilogue";
    if (p.flags & GEMM_OUT_F32) return "fp32 output";
    if (p.b_batch_dim >= 0) return "batched B";
    if (p.alpha != 1.0f) return "alpha != 1";
    if (p.N % 8 != 0) return "N % 8 != 0";
    if ((p.ldo & 7) != 0 || !a16(p.out)) return "output rows not 16-byte aligned";
    if (p.residual != nullptr && ((p.ldr & 7) != 0 || !a16(p.residual))) return "residual rows not 16-byte aligned";
    if (p.bias != nullptr && ((p.bias_stride & 7) != 0 || !a16(p.bias))) return "bias rows not 16-byte aligned";
    return nullptr;
}

long long gemm_splitk_scratch_elems(const GemmProblem& p, int splits) { return static_cast<long long>(splits) * problem_rows(p) * p.N; }

GemmProblem gemm_splitk_partials(const GemmProblem& p, int splits, float* scratch) {
    GemmProblem q = p;
    q.out = scratch;
    q.ldo = p.N;
    q.flags |= GEMM_OUT_F32;
    q.bias = nullptr;
    q.bias_rows = 0;
    q.residual = nullptr;
    q.splits = splits;
    q.split_stride = problem_rows(p) * p.N;
    return q;
}

int gemm_splitk_reduce(const GemmProblem& p, int splits, const float* scratch, cudaStream_t stream) {
    const long long rows = problem_rows(p);
    return splitk_reduce(scratch, splits, rows * p.N, rows, p.N, p.bias, p.bias_rows, p.bias_stride, p.residual, p.ldr,
                         reinterpret_cast<__half*>(p.out), p.ldo, stream);
}

}  // namespace t2v
