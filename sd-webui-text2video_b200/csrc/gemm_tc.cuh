// Implicit-GEMM engine on wgmma + TMA: every dense contraction of the denoiser / VAE (Linear, Conv1d k=1,
// Conv2d 1x1 / 3x3, Conv3d (3,1,1)) is one launch of gemm_tc_kernel.
//
//   D[row, n] = sum_{tap} sum_{k} A[row + tap_offset(tap), k] * W[tap][n][k]   (+ bias, + residual, GEGLU ...)
//
// Activations live channels-last in HBM: A is a [rows, C] fp16 matrix whose rows are the (sample, frame, y, x)
// tokens.  A TMA tensor map of rank 1+nd views the rows as an nd-dimensional grid (e.g. C,w,h,F,B); a "tap" is
// an integer offset in that grid, and TMA's out-of-bounds zero fill IS the convolution's zero padding -- no
// im2col buffer, no transposes.  Weights are packed once as W[tap][N][K] (K-major).
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace t2v {

constexpr int GEMM_BLOCK_M = 128;
constexpr int GEMM_BLOCK_K = 64;     // 64 fp16 = 128 B = one SWIZZLE_128B row
constexpr int GEMM_MAX_TAPS = 9;
constexpr int GEMM_MAX_RDIMS = 4;

enum GemmFlags : int {
    GEMM_GEGLU = 1,        // epilogue: out[:, j] = (acc[:, j] + b) * gelu(acc[:, BN/2 + j] + b)  (weights interleaved per tile)
    GEMM_OUT_F32 = 2,      // store fp32 instead of fp16 (no residual)
    GEMM_LN = 4,           // LayerNorm of the A rows folded into the epilogue: out = rstd_r * (acc - mean_r * colsum_n) + bias32_n
                           //   (weights pre-scaled by gamma; colsum_n = sum_k W'[n,k]; bias32_n = sum_k W[n,k] beta_k + bias_n)
    // switches of t2v_op_gemm (never set by the model code)
    GEMM_DBG_FORCE_BS = 2048,  // t2v_op_gemm only: take the B-stationary variant whenever it is eligible (any K chunk count)
    GEMM_DBG_NO_BS = 4096,     // t2v_op_gemm only: never take it
    GEMM_DBG_SLAB_OUT = 8192,  // t2v_op_gemm only: store through the per-warp slabs even where TMA stores could
};

struct GemmDesc {
    CUtensorMap map_a;               // rank 1 + nd : (K, d0, d1, ...)
    CUtensorMap map_b;               // rank 3      : (K, N, taps | batch)
    CUtensorMap map_o;               // tma_out: rank 1 + nd : (output columns, d0, d1, ...) over `out`
    CUtensorMap map_r;               // tma_out with a residual: the same over `residual`
    int tma_out;                     // 1: fp16 tiles leave through TMA stores from a shared output tile (else per-warp slabs)
    int nd;                          // number of row dims (1..4)
    int dim[GEMM_MAX_RDIMS];         // extent of each row dim (d0 fastest)
    int box[GEMM_MAX_RDIMS];         // rows-box extent per dim; prod(box) <= 128
    int tdim[GEMM_MAX_RDIMS];        // tiles per dim
    int tiles_m, tiles_n;
    int ntaps, k_chunks;
    int8_t tap_off[GEMM_MAX_TAPS][GEMM_MAX_RDIMS];
    int b_batch_dim;                 // >=0: B coordinate 2 = tile origin along that row dim (batched GEMM)
    int a_tx_bytes;                  // bytes one A box load deposits
    int N;                           // valid output columns (GEGLU: of the packed 2x-wide accumulator)
    int flags;
    void* out;
    long long ldo;                   // output row pitch (elements)
    const __half* bias;              // [N] (packed order) or null
    int bias_rows;                   // >0: bias row = global_row / bias_rows (per-sample bias, e.g. time-embedding)
    long long bias_stride;
    const __half* residual;          // [rows, ldr] or null
    long long ldr;
    float alpha;                     // accumulator scale applied before bias (1.0 normally)
    const float2* rowstat;           // GEMM_LN: (mean, rstd) per global row
    const float* colsum;             // GEMM_LN: per packed column
    const float* bias32;             // GEMM_LN: per packed column (replaces `bias`)
    int splits;                      // split-K: work item = (tile, split); each split owns k_per_split k-iterations and
    int k_per_split;                 //   stores its fp32 partial tile at out + split * split_stride (reduced by splitk_reduce)
    long long split_stride;
    int bs_stages;                   // B-stationary variant: depth of the A-only ring (the weight slice of the N-tile is resident)
};

struct GemmProblem {
    const __half* a;
    long long lda;                   // row pitch of A in elements (>= K, multiple of 8)
    int K;                           // channels per tap
    int nd;
    int dim[GEMM_MAX_RDIMS];
    int ntaps;
    int tap_off[GEMM_MAX_TAPS][GEMM_MAX_RDIMS];
    const __half* b;                 // packed [taps or batch][n_alloc][K]
    long long ldb;                   // row pitch of b in elements (0 -> K)
    int n_alloc;                     // allocated rows per tap in b (>= N, allows padding for tiny N)
    int N;
    int b_batch_dim;                 // -1 if none
    int flags;
    void* out;
    long long ldo;
    const __half* bias;
    int bias_rows;
    long long bias_stride;
    const __half* residual;
    long long ldr;
    float alpha;
    int force_bn;                    // 0 = auto
    int force_cg;                    // 0 = auto, 1 / 2 (2: cluster of two M-tiles sharing each B box through TMA multicast)
    const float2* rowstat;           // GEMM_LN operands (see GemmFlags)
    const float* colsum;
    const float* bias32;
    int splits;                      // 0/1 = no split-K; >1: out must be fp32 [splits][rows][ldo], no bias/residual/GEGLU
    long long split_stride;          // elements between split partials
    int force_bs;                    // 0 = auto, 1 = B-stationary if eligible, -1 = never (tests / A-B runs)
    int slab_out;                    // 1 = per-warp slab stores even where TMA stores could (tests)
};

struct GemmPlan {
    GemmDesc desc;
    int bn;
    int cg;                          // 1 = one CTA per tile, 2 = cluster of two CTAs (two M-tiles) that multicast halves of B
    int bs;                          // 1 = B-stationary variant (CTA = one N-tile, walks M-tiles; weights resident in smem)
    int slab;                        // 1 = variant without the output tile (slab stores, one more ring stage; BN 224 / 256)
    int grid;
    int smem;
    double flops;
};

// Builds tensor maps / tile shapes for a problem.  Returns 0 on success.
int gemm_plan(const GemmProblem& p, GemmPlan* plan, int num_sms);
int gemm_launch(const GemmPlan& plan, cudaStream_t stream);

// ---- split-K (fp16 output of a contraction too small to fill the machine): the kernel writes one fp32 partial per split
// into scratch [splits][rows][N], then gemm_splitk_reduce folds them in split order and adds bias and residual.
// Split count the kernel runs for `requested` splits of p: each split owns ceil(kt / requested) of the kt = taps x K-chunk
// iterations and splits that would be left empty are dropped (kt = 30, 7 requested -> 6 splits of 5).  gemm_plan and the
// fix-up pass both take the count from here.
int gemm_split_count(const GemmProblem& p, int requested);
// Why p cannot be split (nullptr if it can): GEGLU, LayerNorm fold, fp32 output, batched B, alpha != 1, N % 8 != 0, or
// output / residual / bias rows the fix-up's 16-byte accesses cannot address.
const char* gemm_splitk_unsupported(const GemmProblem& p);
// fp32 elements the partials of `splits` splits occupy
long long gemm_splitk_scratch_elems(const GemmProblem& p, int splits);
// The partial-sum problem of p: same contraction, fp32 out into scratch, no bias / residual, `splits` = gemm_split_count
GemmProblem gemm_splitk_partials(const GemmProblem& p, int splits, float* scratch);
// Folds the partials gemm_splitk_partials(p, splits, scratch) wrote and applies p's bias (per sample with bias_rows) and
// residual into p.out.
int gemm_splitk_reduce(const GemmProblem& p, int splits, const float* scratch, cudaStream_t stream);
// One-time: cudaFuncSetAttribute for all instantiations + driver entry point lookup.
int gemm_init();
// fp16 tensor map of rank `rank` with SWIZZLE_128B (box[0] = 64 elements); strides_bytes has rank-1 entries (dims 1..)
int tma_encode_f16(CUtensorMap* m, const void* base, int rank, const unsigned long long* dims,
                   const unsigned long long* strides_bytes, const unsigned* box);

}  // namespace t2v
