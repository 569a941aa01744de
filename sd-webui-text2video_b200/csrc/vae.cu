// AutoencoderKL.decode as a pre-planned launch list: post_quant_conv -> ldm Decoder (mid ResnetBlock / single-head
// AttnBlock / ResnetBlock, 4 up levels with nearest-2x + conv) -> norm_out, swish, conv_out.
// Replaces modelscope/t2v_model.py:1646-1649 + ldm.modules.diffusionmodules.model.Decoder (vendored twin:
// videocrafter/lvdm/models/modules/autoencoder_modules.py:484-596) and batches ALL frames of the clip instead of the
// reference's one-frame-per-call loop with a D2H sync per frame (t2v_pipeline.py:329-355).
// Same channels-last token layout and the same wgmma implicit-GEMM engine as the denoiser.
#include "../../include/t2v_b200.h"
#include "runtime.cuh"

#include <cstdio>
#include <cstring>
#include <memory>

namespace t2v {
namespace {

struct VIO {
    __half* z_tok;
    __half* out_tok;
    int out_ld;
};
struct EncIO {
    __half* x_tok;
    __half* out_tok;
    int out_ld;
    int ho, wo;
};

}  // namespace
}  // namespace t2v

using namespace t2v;

struct t2v_vae {
    t2v_vae_config cfg;
    ParamStore params;          // decoder + post_quant_conv (the hot path: missing_params counts these)
    ParamStore enc_params;      // encoder + quant_conv (vid2vid / img2vid latent preparation; optional)
    PlanCache<VIO> plans{3};    // key: "frames,h,w"
    PlanCache<EncIO> enc_plans{3};
    GnWorkspace gn_ws;          // shared by the decoder's and the encoder's plans
};

namespace t2v {
namespace {

// Grows the shared groupnorm workspace; a new pointer drops the plans of both directions, which captured the old one.
bool ensure_gn_ws(t2v_vae* v, size_t need, cudaStream_t stream) {
    if (v->gn_ws.ensure(need, stream)) {
        v->plans.clear(stream);
        v->enc_plans.clear(stream);
    }
    return v->gn_ws.ptr != nullptr;
}

void expect_params(t2v_vae* v) {
    ParamStore& P = v->params;
    const t2v_vae_config& c = v->cfg;
    auto conv = [&](const std::string& p, int o, int i, int k) {
        P.expect(p + ".weight", {o, i, k, k});
        P.expect(p + ".bias", {o});
    };
    auto norm = [&](const std::string& p, int ch) {
        P.expect(p + ".weight", {ch});
        P.expect(p + ".bias", {ch});
    };
    auto resnet = [&](const std::string& p, int ci, int co) {
        norm(p + ".norm1", ci);
        conv(p + ".conv1", co, ci, 3);
        norm(p + ".norm2", co);
        conv(p + ".conv2", co, co, 3);
        if (ci != co) conv(p + ".nin_shortcut", co, ci, 1);
    };
    conv("post_quant_conv", c.z_channels, c.embed_dim, 1);
    int block_in = c.ch * c.ch_mult[c.n_mult - 1];
    conv("decoder.conv_in", block_in, c.z_channels, 3);
    resnet("decoder.mid.block_1", block_in, block_in);
    norm("decoder.mid.attn_1.norm", block_in);
    for (const char* n : {"q", "k", "v", "proj_out"}) conv(std::string("decoder.mid.attn_1.") + n, block_in, block_in, 1);
    resnet("decoder.mid.block_2", block_in, block_in);
    for (int lvl = c.n_mult - 1; lvl >= 0; --lvl) {
        const int block_out = c.ch * c.ch_mult[lvl];
        for (int j = 0; j < c.num_res_blocks + 1; ++j) {
            resnet("decoder.up." + std::to_string(lvl) + ".block." + std::to_string(j), block_in, block_out);
            block_in = block_out;
        }
        if (lvl != 0) conv("decoder.up." + std::to_string(lvl) + ".upsample.conv", block_in, block_in, 3);
    }
    norm("decoder.norm_out", block_in);
    conv("decoder.conv_out", c.out_ch, block_in, 3);
}

// ldm Encoder (autoencoder_modules.py:382-446) + quant_conv (t2v_model.py:1603)
void expect_enc_params(t2v_vae* v) {
    ParamStore& P = v->enc_params;
    const t2v_vae_config& c = v->cfg;
    auto conv = [&](const std::string& p, int o, int i, int k) {
        P.expect(p + ".weight", {o, i, k, k});
        P.expect(p + ".bias", {o});
    };
    auto norm = [&](const std::string& p, int ch) {
        P.expect(p + ".weight", {ch});
        P.expect(p + ".bias", {ch});
    };
    auto resnet = [&](const std::string& p, int ci, int co) {
        norm(p + ".norm1", ci);
        conv(p + ".conv1", co, ci, 3);
        norm(p + ".norm2", co);
        conv(p + ".conv2", co, co, 3);
        if (ci != co) conv(p + ".nin_shortcut", co, ci, 1);
    };
    conv("encoder.conv_in", c.ch, 3, 3);
    int block_in = c.ch;
    for (int lvl = 0; lvl < c.n_mult; ++lvl) {
        const int block_out = c.ch * c.ch_mult[lvl];
        for (int j = 0; j < c.num_res_blocks; ++j) {
            resnet("encoder.down." + std::to_string(lvl) + ".block." + std::to_string(j), block_in, block_out);
            block_in = block_out;
        }
        if (lvl != c.n_mult - 1) conv("encoder.down." + std::to_string(lvl) + ".downsample.conv", block_in, block_in, 3);
    }
    resnet("encoder.mid.block_1", block_in, block_in);
    norm("encoder.mid.attn_1.norm", block_in);
    for (const char* n : {"q", "k", "v", "proj_out"}) conv(std::string("encoder.mid.attn_1.") + n, block_in, block_in, 1);
    resnet("encoder.mid.block_2", block_in, block_in);
    norm("encoder.norm_out", block_in);
    conv("encoder.conv_out", 2 * c.z_channels, block_in, 3);
    conv("quant_conv", 2 * c.embed_dim, 2 * c.z_channels, 1);
}

// ResnetBlock.forward (autoencoder_modules.py:207-228, temb None): x + conv2(swish(GN(conv1(swish(GN(x))))))
Tok resnet(NetCtx& c, const Tok& x, const std::string& p, int co, int hc, int wc) {
    const long long P = static_cast<long long>(hc) * wc;
    Tok a = group_norm(c, x, p + ".norm1", P, 1e-6f, true);
    Tok h = conv3x3(c, a, p + ".conv1.weight", prm(c, p + ".conv1.bias"), 0, 0, co, hc, wc, nullptr);
    c.b->free(a);
    Tok b2 = group_norm(c, h, p + ".norm2", P, 1e-6f, true);
    c.b->free(h);
    Tok skip = x;
    bool own = false;
    if (x.C != co) {
        skip = linear(c, x, prm(c, p + ".nin_shortcut.weight"), co, prm(c, p + ".nin_shortcut.bias"), nullptr);
        own = true;
    }
    Tok y = conv3x3(c, b2, p + ".conv2.weight", prm(c, p + ".conv2.bias"), 0, 0, co, hc, wc, &skip);
    c.b->free(b2);
    if (own) c.b->free(skip);
    return y;
}

// AttnBlock.forward (autoencoder_modules.py:91-116): single head, d = C; per-frame S x S scores through HBM
// (S = h*w <= a few thousand at the latent resolution; 2% of the clip's FLOPs).
Tok attn_block(NetCtx& c, const Tok& x, const std::string& p, int frames, int hc, int wc) {
    const int C = x.C;
    const int S = hc * wc;
    Tok n = group_norm(c, x, p + ".norm", S, 1e-6f, false);
    Tok q = linear(c, n, prm(c, p + ".q.weight"), C, prm(c, p + ".q.bias"), nullptr);
    Tok k = linear(c, n, prm(c, p + ".k.weight"), C, prm(c, p + ".k.bias"), nullptr);
    Tok v = linear(c, n, prm(c, p + ".v.weight"), C, prm(c, p + ".v.bias"), nullptr);
    c.b->free(n);
    // scores[f] = q[f] k[f]^T (fp16, as torch.bmm under autocast), batched over frames
    Tok sc = c.b->alloc(static_cast<long long>(frames) * S, S);
    {
        GemmProblem pr = base_problem(q, C, k.p, S, S, sc);
        pr.nd = 2;
        pr.dim[0] = S;
        pr.dim[1] = frames;
        pr.b_batch_dim = 1;
        c.b->gemm(pr);
    }
    c.b->free(q);
    c.b->free(k);
    Tok pm = c.b->alloc(static_cast<long long>(frames) * S, S);
    {
        const float scale = 1.0f / sqrtf(static_cast<float>(C));
        const Tok s0 = sc;
        c.b->step([=](cudaStream_t st) { return softmax_rows(s0.p, pm.p, s0.rows, S, scale, st); });
    }
    c.b->free(sc);
    Tok vt = c.b->alloc(static_cast<long long>(frames) * C, S);      // V^T per frame: [C, S]
    {
        const Tok v0 = v;
        c.b->step([=](cudaStream_t st) { return transpose_batched(v0.p, vt.p, frames, S, C, st); });
    }
    c.b->free(v);
    Tok o = c.b->alloc(static_cast<long long>(frames) * S, C);
    {
        GemmProblem pr = base_problem(pm, S, vt.p, C, C, o);
        pr.nd = 2;
        pr.dim[0] = S;
        pr.dim[1] = frames;
        pr.b_batch_dim = 1;
        c.b->gemm(pr);
    }
    c.b->free(pm);
    c.b->free(vt);
    Tok y = linear(c, o, prm(c, p + ".proj_out.weight"), C, prm(c, p + ".proj_out.bias"), &x);
    c.b->free(o);
    return y;
}

int build(t2v_vae* v, Plan* plan, Arena* arena, bool dry, cudaStream_t stream, int frames, int h, int w, VIO* io) {
    Builder bld(plan, arena, dry, num_sms());
    NetCtx c{&v->params, &bld, stream, v->gn_ws.ptr};
    const t2v_vae_config& cfg = v->cfg;
    const long long R0 = static_cast<long long>(frames) * h * w;
    const int zpad = round_up(cfg.z_channels, 8);
    Tok z = bld.alloc(R0, zpad);
    io->z_tok = z.p;
    // post_quant_conv 1x1 (t2v_model.py:1647): weights zero-padded to [16][zpad] so the padded channels stay zero
    Tok zq = bld.alloc(R0, zpad);
    {
        const __half* w = w_conv(c, "post_quant_conv.weight", 1, 16, zpad);
        GemmProblem pr = base_problem(z, zpad, w, 16, zpad, zq);
        pr.bias = prm(c, "post_quant_conv.bias");
        bld.gemm(pr);
    }
    int hc = h, wc = w;
    int block_in = cfg.ch * cfg.ch_mult[cfg.n_mult - 1];
    Tok x = conv3x3(c, zq, "decoder.conv_in.weight", prm(c, "decoder.conv_in.bias"), 0, 0, block_in, hc, wc, nullptr);
    bld.free(zq);
    Tok y = resnet(c, x, "decoder.mid.block_1", block_in, hc, wc);
    bld.free(x);
    x = y;
    y = attn_block(c, x, "decoder.mid.attn_1", frames, hc, wc);
    bld.free(x);
    x = y;
    y = resnet(c, x, "decoder.mid.block_2", block_in, hc, wc);
    bld.free(x);
    x = y;
    for (int lvl = cfg.n_mult - 1; lvl >= 0; --lvl) {
        const int block_out = cfg.ch * cfg.ch_mult[lvl];
        for (int j = 0; j < cfg.num_res_blocks + 1; ++j) {
            y = resnet(c, x, "decoder.up." + std::to_string(lvl) + ".block." + std::to_string(j), block_out, hc, wc);
            bld.free(x);
            x = y;
        }
        if (lvl != 0) {
            Tok u = bld.alloc(x.rows * 4, x.C);
            {
                const Tok xx = x;
                const int hh = hc, ww = wc;
                bld.step([=](cudaStream_t s) { return upsample2x(xx.p, u.p, frames, hh, ww, xx.C, s); });
            }
            bld.free(x);
            hc *= 2;
            wc *= 2;
            const std::string up = "decoder.up." + std::to_string(lvl) + ".upsample.conv";
            x = conv3x3(c, u, up + ".weight", prm(c, up + ".bias"), 0, 0, u.C, hc, wc, nullptr);
            bld.free(u);
        }
    }
    Tok g = group_norm(c, x, "decoder.norm_out", static_cast<long long>(hc) * wc, 1e-6f, true);
    bld.free(x);
    Tok o = conv3x3(c, g, "decoder.conv_out.weight", prm(c, "decoder.conv_out.bias"), 0, 0, cfg.out_ch, hc, wc, nullptr, 16);
    bld.free(g);
    io->out_tok = o.p;
    io->out_ld = static_cast<int>(o.ld);
    return bld.error;
}

std::string shape_key(int frames, int h, int w) {
    return std::to_string(frames) + "," + std::to_string(h) + "," + std::to_string(w);
}

PlanCache<VIO>::Entry* get_plan(t2v_vae* v, int frames, int h, int w, cudaStream_t stream) {
    const std::string key = shape_key(frames, h, w);
    if (auto* e = v->plans.find(key, v->params.version())) return e;
    if (!v->params.complete("VAE")) return nullptr;
    const size_t need = std::max(gn_workspace_bytes(h * w, frames, num_sms()), gn_workspace_bytes(h * w * 64, frames, num_sms()));
    if (!ensure_gn_ws(v, need + (1 << 20), stream)) return nullptr;
    return v->plans.build(key, v->params.version(), stream, std::unique_ptr<Plan>(new Plan()), false, "VAE",
                          [&](Plan* p, Arena* a, bool dry, VIO* io) { return build(v, p, a, dry, stream, frames, h, w, io); });
}


// AutoencoderKL.encode up to the moments (t2v_model.py:1640-1644; Encoder.forward autoencoder_modules.py:448-482):
// frames [N,3,H,W] -> tokens -> conv_in -> per level 2 ResnetBlocks (+ Downsample: pad (0,1,0,1), 3x3 stride 2) -> mid
// (ResnetBlock, AttnBlock, ResnetBlock) -> GN + swish -> conv_out -> quant_conv 1x1 -> (mean | logvar) tokens.

int build_enc(t2v_vae* v, Plan* plan, Arena* arena, bool dry, cudaStream_t stream, int frames, int H, int W, EncIO* io) {
    Builder bld(plan, arena, dry, num_sms());
    NetCtx c{&v->enc_params, &bld, stream, v->gn_ws.ptr};
    const t2v_vae_config& cfg = v->cfg;
    int hc = H, wc = W;
    Tok x0 = bld.alloc(static_cast<long long>(frames) * H * W, 8);          // RGB zero-padded to 8 channels
    io->x_tok = x0.p;
    Tok x = conv3x3(c, x0, "encoder.conv_in.weight", prm(c, "encoder.conv_in.bias"), 0, 0, cfg.ch, hc, wc, nullptr);
    int block_in = cfg.ch;
    for (int lvl = 0; lvl < cfg.n_mult; ++lvl) {
        const int block_out = cfg.ch * cfg.ch_mult[lvl];
        for (int j = 0; j < cfg.num_res_blocks; ++j) {
            Tok y = resnet(c, x, "encoder.down." + std::to_string(lvl) + ".block." + std::to_string(j), block_out, hc, wc);
            bld.free(x);
            x = y;
            block_in = block_out;
        }
        if (lvl != cfg.n_mult - 1) {
            const int ho = hc / 2, wo = wc / 2;
            Tok col = bld.alloc(static_cast<long long>(frames) * ho * wo, 9 * x.C);
            {
                const Tok xx = x;
                const int hh = hc, ww = wc;
                bld.step([=](cudaStream_t s) { return im2col_s2(xx.p, col.p, frames, hh, ww, xx.C, s, 0); });
            }
            const std::string dn = "encoder.down." + std::to_string(lvl) + ".downsample.conv";
            const __half* w = w_conv_kmajor(c, dn + ".weight");
            Tok y = linear(c, col, w, block_in, prm(c, dn + ".bias"), nullptr);
            bld.free(col);
            bld.free(x);
            x = y;
            hc = ho;
            wc = wo;
        }
    }
    Tok y = resnet(c, x, "encoder.mid.block_1", block_in, hc, wc);
    bld.free(x);
    x = y;
    y = attn_block(c, x, "encoder.mid.attn_1", frames, hc, wc);
    bld.free(x);
    x = y;
    y = resnet(c, x, "encoder.mid.block_2", block_in, hc, wc);
    bld.free(x);
    x = y;
    Tok g = group_norm(c, x, "encoder.norm_out", static_cast<long long>(hc) * wc, 1e-6f, true);
    bld.free(x);
    const int M = 2 * cfg.z_channels;
    Tok h = conv3x3(c, g, "encoder.conv_out.weight", prm(c, "encoder.conv_out.bias"), 0, 0, M, hc, wc, nullptr, 16);
    bld.free(g);
    Tok mom = bld.alloc(h.rows, 2 * cfg.embed_dim, round_up(2 * cfg.embed_dim, 8));
    {
        const __half* w = w_conv(c, "quant_conv.weight", 1, 16, static_cast<int>(h.ld));
        GemmProblem pr = base_problem(h, static_cast<int>(h.ld), w, 16, 2 * cfg.embed_dim, mom);
        pr.bias = prm(c, "quant_conv.bias");
        bld.gemm(pr);
    }
    bld.free(h);
    io->out_tok = mom.p;
    io->out_ld = static_cast<int>(mom.ld);
    io->ho = hc;
    io->wo = wc;
    return bld.error;
}

PlanCache<EncIO>::Entry* get_enc_plan(t2v_vae* v, int frames, int H, int W, cudaStream_t stream) {
    const std::string key = shape_key(frames, H, W);
    if (auto* e = v->enc_plans.find(key, v->enc_params.version())) return e;
    if (!v->enc_params.complete("VAE encoder")) return nullptr;
    if (!ensure_gn_ws(v, gn_workspace_bytes(H * W, frames, num_sms()) + (1 << 20), stream)) return nullptr;
    return v->enc_plans.build(key, v->enc_params.version(), stream, std::unique_ptr<Plan>(new Plan()), false, "VAE encoder",
                              [&](Plan* p, Arena* a, bool dry, EncIO* io) { return build_enc(v, p, a, dry, stream, frames, H, W, io); });
}

}  // namespace
}  // namespace t2v

extern "C" {

int t2v_vae_create(const t2v_vae_config* cfg, t2v_vae** out) {
    if (!cfg || !out) return -1;
    if (cfg->ch % 32 != 0 || cfg->z_channels > 8 || cfg->out_ch > 8) {
        set_error("unsupported VAE config");
        return -2;
    }
    t2v_vae* v = new t2v_vae();
    v->cfg = *cfg;
    expect_params(v);
    expect_enc_params(v);
    *out = v;
    return 0;
}

void t2v_vae_destroy(t2v_vae* v) { delete v; }

int t2v_vae_set_param(t2v_vae* v, const char* name, const void* data, int dtype, int ndim, const int64_t* shape,
                      void* stream) {
    const bool enc = strncmp(name, "encoder.", 8) == 0 || strncmp(name, "quant_conv.", 11) == 0;
    return (enc ? v->enc_params : v->params).set(name, data, dtype, ndim, shape, reinterpret_cast<cudaStream_t>(stream));
}

int t2v_vae_missing_params(t2v_vae* v, char* name_out, size_t name_cap) { return missing_params_out(v->params, name_out, name_cap); }

// LoRA: a weight lives in the decoder's store or in the encoder's, as t2v_vae_set_param routes it
int t2v_vae_lora_apply(t2v_vae* v, const char* weight_name, const void* up, const void* down, int dtype, int rank, float alpha,
                       void* stream) {
    clear_pending_error("t2v_vae_lora_apply");
    ParamStore& P = v->params.has(weight_name) ? v->params : v->enc_params;
    return P.lora_apply(weight_name, up, down, dtype, rank, alpha, reinterpret_cast<cudaStream_t>(stream));
}

int t2v_vae_lora_restore(t2v_vae* v, const char* weight_name, void* stream) {
    clear_pending_error("t2v_vae_lora_restore");
    ParamStore& P = v->params.has(weight_name) ? v->params : v->enc_params;
    return P.lora_restore(weight_name, reinterpret_cast<cudaStream_t>(stream));
}

int t2v_vae_lora_clear(t2v_vae* v, void* stream) {
    const int rc = v->params.lora_clear(reinterpret_cast<cudaStream_t>(stream));
    return rc != 0 ? rc : v->enc_params.lora_clear(reinterpret_cast<cudaStream_t>(stream));
}

int t2v_vae_lora_merged(t2v_vae* v) { return v->params.merged_count() + v->enc_params.merged_count(); }

int t2v_vae_param_info(t2v_vae* v, int index, char* name_out, size_t name_cap, int64_t* shape_out, int* ndim_out) {
    // decoder-side parameters first, then the encoder's (same state_dict, t2v_model.py:1585-1617)
    const int n_dec = v->params.info(0, nullptr, nullptr);
    const int n_enc = v->enc_params.info(0, nullptr, nullptr);
    if (index < 0 || index >= n_dec + n_enc) return -1;
    if (index < n_dec) param_info_out(v->params, index, name_out, name_cap, shape_out, ndim_out);
    else param_info_out(v->enc_params, index - n_dec, name_out, name_cap, shape_out, ndim_out);
    return n_dec + n_enc;
}

int t2v_vae_decode(t2v_vae* v, const void* z, int z_is_f32, float z_scale, void* out, int out_mode, int B, int F, int h,
                   int w, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const int frames = B * F;
    auto* entry = get_plan(v, frames, h, w, stream);
    if (!entry) return -1;
    const VIO& io = entry->io;
    const int zpad = (v->cfg.z_channels + 7) / 8 * 8;
    int rc = ingest_latent(z, z_is_f32, io.z_tok, zpad, zpad, B, v->cfg.z_channels, F, h, w, z_scale, stream);
    if (rc != 0) return rc;
    rc = run_plan(entry->plan.get(), stream, true);
    if (rc != 0) {
        set_error("VAE launch failed (%d): %s", rc, cudaGetErrorString(cudaGetLastError()));
        return rc;
    }
    const int H = h * 8, W = w * 8;       // 3 upsamples for the 4-level decoder
    int up = 1;
    for (int i = 1; i < v->cfg.n_mult; ++i) up *= 2;
    const int Ho = h * up, Wo = w * up;
    (void)H;
    (void)W;
    if (out_mode == 1)
        return frames_to_u8(io.out_tok, io.out_ld, reinterpret_cast<uint8_t*>(out), static_cast<long long>(frames) * Ho * Wo,
                            stream);
    return frames_to_f32_nchw(io.out_tok, io.out_ld, reinterpret_cast<float*>(out), frames, Ho, Wo, stream);
}

int t2v_vae_encode(t2v_vae* v, const void* x, int x_is_f32, void* moments_out, int N, int H, int W, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    int down = 1;
    for (int i = 1; i < v->cfg.n_mult; ++i) down *= 2;
    if (N < 1 || H % down != 0 || W % down != 0) {
        set_error("t2v_vae_encode: H and W must be multiples of %d (got %d x %d)", down, H, W);
        return -3;
    }
    auto* entry = get_enc_plan(v, N, H, W, stream);
    if (!entry) return -1;
    const EncIO& io = entry->io;
    int rc = ingest_latent(x, x_is_f32, io.x_tok, 8, 8, N, 3, 1, H, W, 1.0f, stream);
    if (rc != 0) return rc;
    rc = run_plan(entry->plan.get(), stream, true);
    if (rc != 0) {
        set_error("VAE encoder launch failed (%d): %s", rc, cudaGetErrorString(cudaGetLastError()));
        return rc;
    }
    return egress_latent(io.out_tok, io.out_ld, moments_out, 1, N, 2 * v->cfg.embed_dim, 1, io.ho, io.wo, stream);
}

double t2v_vae_flops(t2v_vae* v, int nframes, int h, int w) {
    VIO io;
    double flops = 0.0;
    if (dry_build(nullptr, false, [&](Plan* p, Arena* a, bool dry) { return build(v, p, a, dry, nullptr, nframes, h, w, &io); }, &flops) < 0)
        return -1.0;
    return flops;
}

}  // extern "C"
