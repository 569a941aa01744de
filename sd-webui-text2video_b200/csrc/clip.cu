// OpenCLIP ViT-H-14 text tower as a pre-planned launch list -- the step right before the denoising loop (SURVEY.md 8 f1).
// Replaces FrozenOpenCLIPEmbedder.encode_with_transformer (modelscope/clip_hardcode.py:112-119, :269-274) on top of
// open_clip's TextTransformer: token embedding + positional embedding, `layers_run` pre-LN residual attention blocks
// (nn.MultiheadAttention with the causal mask, GELU MLP; the reference stops one block early: layer = 'penultimate'),
// ln_final.  open_clip is NOT under /root/reference (pip dependency, unpinned by the reference's requirements.txt): the
// architecture restated here is open_clip's published ResidualAttentionBlock, pinned in tests against torch's own
// nn.MultiheadAttention / nn.LayerNorm modules.
//
// Same engine as the denoiser: LayerNorm folded into the consuming wgmma GEMM, residual adds in the GEMM epilogue; the
// 77-token causal attention and the GELU are small dedicated kernels (the tower runs once per prompt: 2 x 77 rows).
//
// arch = 1 is the OpenAI CLIP ViT-L/14 text model of VideoCrafter's FrozenCLIPEmbedder (videocrafter/lvdm/models/modules/
// condition_modules.py:15-40: transformers' CLIPTextModel, `last_hidden_state`).  Same block structure with transformers'
// parameter names, separate q / k / v projections (fused here into one [q|k|v] weight and bias, so the block keeps one
// LayerNorm-folded projection GEMM), quick_gelu instead of GELU, every layer, then final_layer_norm.
#include "../../include/t2v_b200.h"
#include "runtime.cuh"

#include <cmath>
#include <cstdio>
#include <cstring>
#include <memory>

namespace t2v {
namespace {

struct ClipIO {
    int* tokens;        // token staging [B * L]
    __half* out;        // output tokens [B * L, width]
};

}  // namespace
}  // namespace t2v

using namespace t2v;

struct t2v_clip {
    t2v_clip_config cfg;
    ParamStore params;
    PlanCache<ClipIO> plans{4};       // key: batch
};

namespace t2v {
namespace {

// x[b, l, :] = token_embedding[tokens[b, l], :] + positional_embedding[l, :]
__global__ void clip_embed_kernel(const int* __restrict__ tokens, const __half* __restrict__ emb, const __half* __restrict__ pos,
                                  __half* __restrict__ x, int rows, int L, int W, int vocab) {
    const int W8 = W >> 3;
    const long long n = static_cast<long long>(rows) * W8;
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        const int r = static_cast<int>(i / W8), vc = static_cast<int>(i - static_cast<long long>(r) * W8);
        int tok = tokens[r];
        tok = tok < 0 ? 0 : (tok >= vocab ? vocab - 1 : tok);
        const uint4 e = __ldg(reinterpret_cast<const uint4*>(emb + static_cast<long long>(tok) * W + vc * 8));
        const uint4 p = __ldg(reinterpret_cast<const uint4*>(pos + static_cast<long long>(r % L) * W + vc * 8));
        const __half2* eh = reinterpret_cast<const __half2*>(&e);
        const __half2* ph = reinterpret_cast<const __half2*>(&p);
        uint4 o;
        __half2* oh = reinterpret_cast<__half2*>(&o);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 a = __half22float2(eh[k]), b = __half22float2(ph[k]);
            oh[k] = __floats2half2_rn(a.x + b.x, a.y + b.y);
        }
        *reinterpret_cast<uint4*>(x + static_cast<long long>(r) * W + vc * 8) = o;
    }
}

// y = x * Phi(x) (nn.GELU, erf form), in place on [rows, C] fp16
__global__ void gelu_kernel(__half* __restrict__ x, long long n8) {
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n8; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        uint4 v = reinterpret_cast<uint4*>(x)[i];
        __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 f = __half22float2(h[k]);
            h[k] = __floats2half2_rn(0.5f * f.x * (1.0f + erff(f.x * 0.70710678118654752440f)),
                                     0.5f * f.y * (1.0f + erff(f.y * 0.70710678118654752440f)));
        }
        reinterpret_cast<uint4*>(x)[i] = v;
    }
}

// y = x * sigmoid(1.702 x) (transformers' quick_gelu, CLIP ViT-L/14), in place on [rows, C] fp16; fp32 math, one rounding
__global__ void quick_gelu_kernel(__half* __restrict__ x, long long n8) {
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n8; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        uint4 v = reinterpret_cast<uint4*>(x)[i];
        __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 f = __half22float2(h[k]);
            h[k] = __floats2half2_rn(f.x / (1.0f + expf(-1.702f * f.x)), f.y / (1.0f + expf(-1.702f * f.y)));
        }
        reinterpret_cast<uint4*>(x)[i] = v;
    }
}

// Causal self-attention over one short sequence per (sample, head): softmax(q k^T / sqrt(d) + causal mask) v, d = 64,
// L <= 128.  qkv [rows, 3W] as nn.MultiheadAttention's in_proj lays it out (q | k | v, head h at columns h*64 of each part).
// One block per (sample, head): K and V of the head in shared memory (rows padded to 66 halves: conflict-free column reads),
// one warp per query row; lanes own keys l, l+32, ... for the scores and output channels l, l+32 for P V.
constexpr int kClipD = 64;
__global__ void __launch_bounds__(128) clip_attention_kernel(const __half* __restrict__ qkv, __half* __restrict__ o, int L, int W, int heads) {
    extern __shared__ __half sm_kv[];
    const int b = blockIdx.x / heads, hd = blockIdx.x % heads;
    __half* sk = sm_kv;                         // [L][66]
    __half* sv = sm_kv + L * 66;                // [L][66]
    __shared__ float sq[4][kClipD];
    __shared__ float sp[4][128];
    const long long row0 = static_cast<long long>(b) * L;
    const int ld = 3 * W;
    for (int i = threadIdx.x; i < L * (kClipD / 2); i += blockDim.x) {
        const int r = i / (kClipD / 2), c2 = i % (kClipD / 2);
        const __half2 kk = *reinterpret_cast<const __half2*>(qkv + (row0 + r) * ld + W + hd * kClipD + c2 * 2);
        const __half2 vv = *reinterpret_cast<const __half2*>(qkv + (row0 + r) * ld + 2 * W + hd * kClipD + c2 * 2);
        *reinterpret_cast<__half2*>(sk + r * 66 + c2 * 2) = kk;
        *reinterpret_cast<__half2*>(sv + r * 66 + c2 * 2) = vv;
    }
    __syncthreads();
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float scale = 0.125f;                 // 64^-0.5
    for (int qi = warp; qi < L; qi += 4) {
        const __half* qp = qkv + (row0 + qi) * ld + hd * kClipD;
        sq[warp][lane] = __half2float(qp[lane]) * scale;             // nn.MultiheadAttention scales q before q k^T
        sq[warp][lane + 32] = __half2float(qp[lane + 32]) * scale;
        __syncwarp();
        float s[4];
        float mx = -INFINITY;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int key = lane + 32 * j;
            s[j] = -INFINITY;
            if (key <= qi && key < L) {                               // causal: keys up to and including the query position
                float acc = 0.f;
                for (int d = 0; d < kClipD; ++d) acc = fmaf(sq[warp][d], __half2float(sk[key * 66 + d]), acc);
                s[j] = acc;
            }
            mx = fmaxf(mx, s[j]);
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
        float sum = 0.f;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float e = s[j] == -INFINITY ? 0.f : __expf(s[j] - mx);
            s[j] = e;
            sum += e;
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
        const float inv = 1.0f / sum;
#pragma unroll
        for (int j = 0; j < 4; ++j) sp[warp][lane + 32 * j] = s[j] * inv;
        __syncwarp();
        float o0 = 0.f, o1 = 0.f;
        for (int key = 0; key <= qi; ++key) {
            const float p = sp[warp][key];
            o0 = fmaf(p, __half2float(sv[key * 66 + lane]), o0);
            o1 = fmaf(p, __half2float(sv[key * 66 + lane + 32]), o1);
        }
        __half* op = o + (row0 + qi) * W + hd * kClipD;
        op[lane] = __float2half_rn(o0);
        op[lane + 32] = __float2half_rn(o1);
        __syncwarp();
    }
}

// arch 1: transformers CLIPTextModel names (relative to the CLIPTextModel)
const char* const kHfEmb = "text_model.embeddings.token_embedding.weight";
const char* const kHfPos = "text_model.embeddings.position_embedding.weight";
const char* const kHfFinal = "text_model.final_layer_norm";
std::string hf_layer(int i) { return "text_model.encoder.layers." + std::to_string(i); }

void expect_params_hf(t2v_clip* m) {
    ParamStore& P = m->params;
    const t2v_clip_config& c = m->cfg;
    P.expect(kHfEmb, {c.vocab, c.width});
    P.expect(kHfPos, {c.context, c.width});
    for (int i = 0; i < c.layers_run; ++i) {
        const std::string p = hf_layer(i);
        for (const char* ln : {".layer_norm1", ".layer_norm2"}) {
            P.expect(p + ln + ".weight", {c.width});
            P.expect(p + ln + ".bias", {c.width});
        }
        for (const char* proj : {".self_attn.q_proj", ".self_attn.k_proj", ".self_attn.v_proj", ".self_attn.out_proj"}) {
            P.expect(p + proj + ".weight", {c.width, c.width});
            P.expect(p + proj + ".bias", {c.width});
        }
        P.expect(p + ".mlp.fc1.weight", {4 * c.width, c.width});
        P.expect(p + ".mlp.fc1.bias", {4 * c.width});
        P.expect(p + ".mlp.fc2.weight", {c.width, 4 * c.width});
        P.expect(p + ".mlp.fc2.bias", {c.width});
    }
    P.expect(std::string(kHfFinal) + ".weight", {c.width});
    P.expect(std::string(kHfFinal) + ".bias", {c.width});
}

void expect_params(t2v_clip* m) {
    if (m->cfg.arch == 1) {
        expect_params_hf(m);
        return;
    }
    ParamStore& P = m->params;
    const t2v_clip_config& c = m->cfg;
    P.expect("token_embedding.weight", {c.vocab, c.width});
    P.expect("positional_embedding", {c.context, c.width});
    for (int i = 0; i < c.layers_run; ++i) {
        const std::string p = "transformer.resblocks." + std::to_string(i);
        P.expect(p + ".ln_1.weight", {c.width});
        P.expect(p + ".ln_1.bias", {c.width});
        P.expect(p + ".attn.in_proj_weight", {3 * c.width, c.width});
        P.expect(p + ".attn.in_proj_bias", {3 * c.width});
        P.expect(p + ".attn.out_proj.weight", {c.width, c.width});
        P.expect(p + ".attn.out_proj.bias", {c.width});
        P.expect(p + ".ln_2.weight", {c.width});
        P.expect(p + ".ln_2.bias", {c.width});
        P.expect(p + ".mlp.c_fc.weight", {4 * c.width, c.width});
        P.expect(p + ".mlp.c_fc.bias", {4 * c.width});
        P.expect(p + ".mlp.c_proj.weight", {c.width, 4 * c.width});
        P.expect(p + ".mlp.c_proj.bias", {c.width});
    }
    P.expect("ln_final.weight", {c.width});
    P.expect("ln_final.bias", {c.width});
}

int build(t2v_clip* m, Plan* plan, Arena* arena, bool dry, cudaStream_t stream, int B, ClipIO* io) {
    Builder bld(plan, arena, dry, num_sms());
    NetCtx c{&m->params, &bld, stream, nullptr};
    const t2v_clip_config& cfg = m->cfg;
    const bool hf = cfg.arch == 1;
    const int L = cfg.context, W = cfg.width, heads = cfg.heads;
    const long long R = static_cast<long long>(B) * L;
    int* tokens = reinterpret_cast<int*>(bld.alloc_bytes(static_cast<size_t>(R) * sizeof(int)));
    io->tokens = tokens;
    Tok x = bld.alloc(R, W);
    {
        const __half* emb = prm(c, hf ? kHfEmb : "token_embedding.weight");
        const __half* pos = prm(c, hf ? kHfPos : "positional_embedding");
        const Tok xx = x;
        const int vocab = cfg.vocab;
        bld.step([=](cudaStream_t s) {
            clip_embed_kernel<<<dim3(static_cast<unsigned>((R * (W / 8) + 255) / 256)), dim3(256), 0, s>>>(tokens, emb, pos, xx.p,
                                                                                                           static_cast<int>(R), L, W, vocab);
            return launch_status("clip launch");
        }, 1, STEP_OTHER, 0.0, "clip embed");
    }
    // per-layer names: open_clip's ResidualAttentionBlock (arch 0) or transformers' CLIPEncoderLayer (arch 1)
    const std::string out_proj = hf ? ".self_attn.out_proj" : ".attn.out_proj";
    const std::string ln2 = hf ? ".layer_norm2" : ".ln_2", fc1 = hf ? ".mlp.fc1" : ".mlp.c_fc", fc2 = hf ? ".mlp.fc2" : ".mlp.c_proj";
    void (*act)(__half*, long long) = hf ? quick_gelu_kernel : gelu_kernel;
    const char* act_label = hf ? "clip quick_gelu" : "clip gelu";
    for (int i = 0; i < cfg.layers_run; ++i) {
        const std::string p = hf ? hf_layer(i) : "transformer.resblocks." + std::to_string(i);
        // x = x + out_proj(attention(in_proj(ln_1(x))))
        Tok qkv;
        if (hf) {       // q / k / v with their biases, concatenated once into one [3W, W] weight and one [3W] bias (cached)
            const std::string a = p + ".self_attn.";
            const __half* wqkv = w_cat(c, {a + "q_proj.weight", a + "k_proj.weight", a + "v_proj.weight"});
            const __half* bqkv = w_cat(c, {a + "q_proj.bias", a + "k_proj.bias", a + "v_proj.bias"});
            qkv = ln_linear(c, x, p + ".layer_norm1", a + "qkv", wqkv, bqkv, 3 * W, nullptr);
        } else {
            qkv = ln_linear(c, x, p + ".ln_1", p + ".attn.in_proj", prm(c, p + ".attn.in_proj_weight"), prm(c, p + ".attn.in_proj_bias"),
                            3 * W, nullptr);
        }
        Tok o = bld.alloc(R, W);
        {
            const Tok q = qkv, oo = o;
            bld.step([=](cudaStream_t s) { return clip_attention(q.p, oo.p, B, L, W, heads, s); }, 1, STEP_ATTN,
                     4.0 * B * heads * static_cast<double>(L) * L * kClipD / 2, "clip causal attention");
        }
        bld.free(qkv);
        Tok y = linear(c, o, prm(c, p + out_proj + ".weight"), W, prm(c, p + out_proj + ".bias"), &x);
        bld.free(o);
        bld.free(x);
        x = y;
        // x = x + c_proj(gelu(c_fc(ln_2(x))))       (arch 1: x + fc2(quick_gelu(fc1(layer_norm2(x)))))
        Tok h = ln_linear(c, x, p + ln2, p + fc1, prm(c, p + fc1 + ".weight"), prm(c, p + fc1 + ".bias"), 4 * W, nullptr);
        {
            const Tok hh = h;
            const long long n8 = R * (4 * W) / 8;
            bld.step([=](cudaStream_t s) {
                act<<<dim3(static_cast<unsigned>((n8 + 255) / 256)), dim3(256), 0, s>>>(hh.p, n8);
                return launch_status("clip launch");
            }, 1, STEP_OTHER, 0.0, act_label);
        }
        Tok y2 = linear(c, h, prm(c, p + fc2 + ".weight"), W, prm(c, p + fc2 + ".bias"), &x);
        bld.free(h);
        bld.free(x);
        x = y2;
    }
    Tok z = layer_norm(c, x, hf ? kHfFinal : "ln_final");
    bld.free(x);
    io->out = z.p;
    return bld.error;
}

PlanCache<ClipIO>::Entry* get_plan(t2v_clip* m, int B, cudaStream_t stream) {
    const std::string key = std::to_string(B);
    if (auto* e = m->plans.find(key, m->params.version())) return e;
    if (!m->params.complete("CLIP text tower")) return nullptr;
    return m->plans.build(key, m->params.version(), stream, std::unique_ptr<Plan>(new Plan()), false, "CLIP",
                          [&](Plan* p, Arena* a, bool dry, ClipIO* io) { return build(m, p, a, dry, stream, B, io); });
}

__global__ void clip_out_kernel(const __half* __restrict__ z, void* __restrict__ out, int out_is_f32, long long n) {
    for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
        if (out_is_f32) reinterpret_cast<float*>(out)[i] = __half2float(z[i]);
        else reinterpret_cast<__half*>(out)[i] = z[i];
    }
}

}  // namespace

int clip_attention(const __half* qkv, __half* o, int B, int L, int W, int heads, cudaStream_t stream) {
    if (B < 1 || heads < 1 || W % kClipD != 0 || W / heads != kClipD || L < 1 || L > 128) {
        set_error("clip_attention: needs W %% 64 == 0, W / heads == 64, 1 <= L <= 128 (B %d, L %d, W %d, heads %d)", B, L, W, heads);
        return -1;
    }
    if (reinterpret_cast<uintptr_t>(qkv) & 3) {        // K and V are read as __half2
        set_error("clip_attention: qkv must be 4-byte aligned");
        return -1;
    }
    const size_t smem = static_cast<size_t>(2) * L * 66 * sizeof(__half);
    clip_attention_kernel<<<dim3(static_cast<unsigned>(B * heads)), dim3(128), smem, stream>>>(qkv, o, L, W, heads);
    return launch_status("clip launch");
}

}  // namespace t2v

extern "C" {

int t2v_op_clip_attention(const void* qkv, void* o, int B, int L, int W, int heads, void* stream) {
    return clip_attention(reinterpret_cast<const __half*>(qkv), reinterpret_cast<__half*>(o), B, L, W, heads,
                          reinterpret_cast<cudaStream_t>(stream));
}

int t2v_clip_create(const t2v_clip_config* cfg, t2v_clip** out) {
    if (!cfg || !out) return -1;
    if (cfg->width % 64 != 0 || cfg->width / cfg->heads != 64 || cfg->context > 128 || cfg->layers_run < 1 || cfg->vocab < 1) {
        set_error("CLIP text tower: head width must be 64 (width / heads), context <= 128");
        return -2;
    }
    if (cfg->arch != 0 && cfg->arch != 1) {
        set_error("CLIP text tower: arch %d (0: OpenCLIP ViT-H-14, 1: transformers CLIPTextModel)", cfg->arch);
        return -2;
    }
    t2v_clip* m = new t2v_clip();
    m->cfg = *cfg;
    expect_params(m);
    *out = m;
    return 0;
}

void t2v_clip_destroy(t2v_clip* m) { delete m; }

int t2v_clip_set_param(t2v_clip* m, const char* name, const void* data, int dtype, int ndim, const int64_t* shape, void* stream) {
    return m->params.set(name, data, dtype, ndim, shape, reinterpret_cast<cudaStream_t>(stream));
}

int t2v_clip_param_info(t2v_clip* m, int index, char* name_out, size_t name_cap, int64_t* shape_out, int* ndim_out) {
    return param_info_out(m->params, index, name_out, name_cap, shape_out, ndim_out);
}

int t2v_clip_lora_apply(t2v_clip* m, const char* weight_name, const void* up, const void* down, int dtype, int rank, float alpha,
                        void* stream) {
    clear_pending_error("t2v_clip_lora_apply");
    return m->params.lora_apply(weight_name, up, down, dtype, rank, alpha, reinterpret_cast<cudaStream_t>(stream));
}

int t2v_clip_lora_restore(t2v_clip* m, const char* weight_name, void* stream) {
    clear_pending_error("t2v_clip_lora_restore");
    return m->params.lora_restore(weight_name, reinterpret_cast<cudaStream_t>(stream));
}

int t2v_clip_lora_clear(t2v_clip* m, void* stream) { return m->params.lora_clear(reinterpret_cast<cudaStream_t>(stream)); }

int t2v_clip_lora_merged(t2v_clip* m) { return m->params.merged_count(); }

int t2v_clip_encode(t2v_clip* m, const int* tokens, void* out, int out_is_f32, int B, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    auto* entry = get_plan(m, B, stream);
    if (!entry) return -1;
    const ClipIO& io = entry->io;
    const long long R = static_cast<long long>(B) * m->cfg.context;
    cudaMemcpyAsync(io.tokens, tokens, static_cast<size_t>(R) * sizeof(int), cudaMemcpyDeviceToDevice, stream);
    const int rc = run_plan(entry->plan.get(), stream, true);
    if (rc != 0) {
        set_error("CLIP launch failed (%d): %s", rc, cudaGetErrorString(cudaGetLastError()));
        return rc;
    }
    const long long n = R * m->cfg.width;
    clip_out_kernel<<<static_cast<unsigned>((n + 255) / 256 > 4096 ? 4096 : (n + 255) / 256), 256, 0, stream>>>(io.out, out, out_is_f32, n);
    return launch_status("clip launch");
}

}  // extern "C"
