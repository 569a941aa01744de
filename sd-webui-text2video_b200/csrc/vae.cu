// AutoencoderKL.decode as a pre-planned launch list: post_quant_conv -> ldm Decoder (mid ResnetBlock / single-head
// AttnBlock / ResnetBlock, 4 up levels with nearest-2x + conv) -> norm_out, swish, conv_out.
// Replaces modelscope/t2v_model.py:1646-1649 + ldm.modules.diffusionmodules.model.Decoder (vendored twin:
// videocrafter/lvdm/models/modules/autoencoder_modules.py:484-596) and batches ALL frames of the clip instead of the
// reference's one-frame-per-call loop with a D2H sync per frame (t2v_pipeline.py:329-355).
// Same channels-last token layout and the same wgmma implicit-GEMM engine as the denoiser.
#include "../../include/t2v_b200.h"
#include "runtime.cuh"

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <memory>
#include <vector>

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
    size_t budget = 0;          // plan bytes (arena + GroupNorm workspace) one direction may hold; 0: automatic
    int last_chunk[2] = {0, 0}, last_n_chunks[2] = {0, 0};      // how the last decode [0] / encode [1] was split
    bool taps_enabled = false;  // plans built meanwhile keep every block's output (t2v_vae_enable_taps)
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

// Block outputs a plan keeps for the parity tests (t2v_vae_read_tap).  With taps on, a tapped activation is recorded under
// the reference module's name and never freed, so the arena cannot reuse its bytes; the dry pass makes the same choices,
// so plan_bytes and the chunking policy see the larger plan.  With taps off, keep() records nothing and release() frees.
struct Taps {
    Plan* plan;
    Builder* b;
    bool on;
    std::vector<const __half*> kept;
    void keep(const std::string& name, const Tok& t, int h, int w) {
        if (!on) return;
        kept.push_back(t.p);
        if (!b->dry()) plan->taps[name] = {t, {h, w}};
    }
    void release(const Tok& t) {
        if (std::find(kept.begin(), kept.end(), t.p) == kept.end()) b->free(t);
    }
};

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
    Taps taps{plan, &bld, v->taps_enabled};
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
    taps.keep("decoder.conv_in", x, hc, wc);
    Tok y = resnet(c, x, "decoder.mid.block_1", block_in, hc, wc);
    taps.release(x);
    x = y;
    taps.keep("decoder.mid.block_1", x, hc, wc);
    y = attn_block(c, x, "decoder.mid.attn_1", frames, hc, wc);
    taps.release(x);
    x = y;
    taps.keep("decoder.mid.attn_1", x, hc, wc);
    y = resnet(c, x, "decoder.mid.block_2", block_in, hc, wc);
    taps.release(x);
    x = y;
    taps.keep("decoder.mid.block_2", x, hc, wc);
    for (int lvl = cfg.n_mult - 1; lvl >= 0; --lvl) {
        const int block_out = cfg.ch * cfg.ch_mult[lvl];
        for (int j = 0; j < cfg.num_res_blocks + 1; ++j) {
            y = resnet(c, x, "decoder.up." + std::to_string(lvl) + ".block." + std::to_string(j), block_out, hc, wc);
            taps.release(x);
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
        taps.keep("decoder.up." + std::to_string(lvl), x, hc, wc);
    }
    Tok g = group_norm(c, x, "decoder.norm_out", static_cast<long long>(hc) * wc, 1e-6f, true);
    taps.release(x);
    taps.keep("decoder.norm_out", g, hc, wc);
    Tok o = conv3x3(c, g, "decoder.conv_out.weight", prm(c, "decoder.conv_out.bias"), 0, 0, cfg.out_ch, hc, wc, nullptr, 16);
    taps.release(g);
    io->out_tok = o.p;
    io->out_ld = static_cast<int>(o.ld);
    return bld.error;
}

std::string shape_key(int frames, int h, int w) {
    return std::to_string(frames) + "," + std::to_string(h) + "," + std::to_string(w);
}

// GroupNorm workspace the decoder's / the encoder's plan of this shape needs (largest and smallest resolution, + 1 MB)
size_t dec_gn_need(int frames, int h, int w) {
    return std::max(gn_workspace_bytes(h * w, frames, num_sms()), gn_workspace_bytes(h * w * 64, frames, num_sms())) + (1 << 20);
}
size_t enc_gn_need(int frames, int H, int W) { return gn_workspace_bytes(H * W, frames, num_sms()) + (1 << 20); }

PlanCache<VIO>::Entry* get_plan(t2v_vae* v, int frames, int h, int w, cudaStream_t stream) {
    const std::string key = shape_key(frames, h, w);
    if (auto* e = v->plans.find(key, v->params.version())) return e;
    if (!v->params.complete("VAE")) return nullptr;
    if (!ensure_gn_ws(v, dec_gn_need(frames, h, w), stream)) return nullptr;
    return v->plans.build(key, v->params.version(), stream, std::unique_ptr<Plan>(new Plan()), false, "VAE",
                          [&](Plan* p, Arena* a, bool dry, VIO* io) { return build(v, p, a, dry, stream, frames, h, w, io); });
}


// AutoencoderKL.encode up to the moments (t2v_model.py:1640-1644; Encoder.forward autoencoder_modules.py:448-482):
// frames [N,3,H,W] -> tokens -> conv_in -> per level 2 ResnetBlocks (+ Downsample: pad (0,1,0,1), 3x3 stride 2) -> mid
// (ResnetBlock, AttnBlock, ResnetBlock) -> GN + swish -> conv_out -> quant_conv 1x1 -> (mean | logvar) tokens.

int build_enc(t2v_vae* v, Plan* plan, Arena* arena, bool dry, cudaStream_t stream, int frames, int H, int W, EncIO* io) {
    Builder bld(plan, arena, dry, num_sms());
    NetCtx c{&v->enc_params, &bld, stream, v->gn_ws.ptr};
    Taps taps{plan, &bld, v->taps_enabled};
    const t2v_vae_config& cfg = v->cfg;
    int hc = H, wc = W;
    Tok x0 = bld.alloc(static_cast<long long>(frames) * H * W, 8);          // RGB zero-padded to 8 channels
    io->x_tok = x0.p;
    Tok x = conv3x3(c, x0, "encoder.conv_in.weight", prm(c, "encoder.conv_in.bias"), 0, 0, cfg.ch, hc, wc, nullptr);
    taps.keep("encoder.conv_in", x, hc, wc);
    int block_in = cfg.ch;
    for (int lvl = 0; lvl < cfg.n_mult; ++lvl) {
        const int block_out = cfg.ch * cfg.ch_mult[lvl];
        for (int j = 0; j < cfg.num_res_blocks; ++j) {
            Tok y = resnet(c, x, "encoder.down." + std::to_string(lvl) + ".block." + std::to_string(j), block_out, hc, wc);
            taps.release(x);
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
            taps.release(x);
            x = y;
            hc = ho;
            wc = wo;
        }
        taps.keep("encoder.down." + std::to_string(lvl), x, hc, wc);
    }
    Tok y = resnet(c, x, "encoder.mid.block_1", block_in, hc, wc);
    taps.release(x);
    x = y;
    taps.keep("encoder.mid.block_1", x, hc, wc);
    y = attn_block(c, x, "encoder.mid.attn_1", frames, hc, wc);
    taps.release(x);
    x = y;
    taps.keep("encoder.mid.attn_1", x, hc, wc);
    y = resnet(c, x, "encoder.mid.block_2", block_in, hc, wc);
    taps.release(x);
    x = y;
    taps.keep("encoder.mid.block_2", x, hc, wc);
    Tok g = group_norm(c, x, "encoder.norm_out", static_cast<long long>(hc) * wc, 1e-6f, true);
    taps.release(x);
    taps.keep("encoder.norm_out", g, hc, wc);
    const int M = 2 * cfg.z_channels;
    Tok h = conv3x3(c, g, "encoder.conv_out.weight", prm(c, "encoder.conv_out.bias"), 0, 0, M, hc, wc, nullptr, 16);
    taps.release(g);
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
    if (!ensure_gn_ws(v, enc_gn_need(frames, H, W), stream)) return nullptr;
    return v->enc_plans.build(key, v->enc_params.version(), stream, std::unique_ptr<Plan>(new Plan()), false, "VAE encoder",
                              [&](Plan* p, Arena* a, bool dry, EncIO* io) { return build_enc(v, p, a, dry, stream, frames, H, W, io); });
}

// ---------------------------------------------------------------------------------------------- frame chunking
// A plan's arena grows linearly with the frame count (0.83 GB per 576 x 1024 decoded frame), so a long or large clip may not
// fit the device as one plan.  Every op of the decoder and the encoder is per frame, so the clip can run as consecutive
// frame ranges instead, each through a plan of that many frames.  Chunking starts only where the whole-clip plan does not
// fit: a clip that fits runs exactly as before.
enum { DEC = 0, ENC = 1 };

// Automatic budget: free device memory, plus what this direction's cached plans and the GroupNorm workspace already hold
// (both are dropped or regrown to make room), minus this margin.  The margin covers what a plan build allocates outside its
// arena: the packed weight copies made on the first build (~100 MB for the SD VAE's decoder in fp16), the instantiated
// CUDA graph and the 2 MB rounding of each allocation, with room left for the caller's own small allocations meanwhile.
constexpr size_t kBudgetMargin = size_t(512) << 20;

// Bytes a plan of `frames` frames would allocate: its activation slab (*arena) and the GroupNorm workspace it needs (*gn).
// Host only (the dry pass).  h, w are what the entry point takes: the latent's for decode, the image's for encode.
int plan_bytes(t2v_vae* v, int dir, int frames, int h, int w, size_t* arena, size_t* gn) {
    long long peak;
    if (dir == DEC) {
        VIO io;
        peak = dry_build(nullptr, false, [&](Plan* p, Arena* a, bool dry) { return build(v, p, a, dry, nullptr, frames, h, w, &io); });
        *gn = dec_gn_need(frames, h, w);
    } else {
        EncIO io;
        peak = dry_build(nullptr, false, [&](Plan* p, Arena* a, bool dry) { return build_enc(v, p, a, dry, nullptr, frames, h, w, &io); });
        *gn = enc_gn_need(frames, h, w);
    }
    if (peak < 0) return -1;
    *arena = plan_slab_bytes(peak);
    return 0;
}

// The largest n <= frames whose plan (arena + GroupNorm workspace) fits `budget`, found by bisection (plan bytes grow with
// the frame count).  Returns 0 with *n set; -4 if not even one frame fits (*one_frame = its plan bytes, error set); -1 if
// the dry pass failed.
int choose_chunk(t2v_vae* v, int dir, int frames, int h, int w, size_t budget, int* n, size_t* one_frame) {
    auto bytes = [&](int f, size_t* out) {
        size_t a = 0, g = 0;
        if (plan_bytes(v, dir, f, h, w, &a, &g) != 0) return false;
        *out = a + g;
        return true;
    };
    size_t b = 0;
    if (!bytes(frames, &b)) return -1;
    if (b <= budget) {
        *n = frames;
        return 0;
    }
    if (!bytes(1, one_frame)) return -1;
    if (*one_frame > budget) {
        set_error("VAE %s of %d frames of %d x %d %s: a one-frame plan needs %.1f MB, more than the memory budget of %.1f MB",
                  dir == DEC ? "decode" : "encode", frames, h, w, dir == DEC ? "latents" : "pixels", *one_frame / 1048576.0,
                  budget / 1048576.0);
        return -4;
    }
    int lo = 1, hi = frames;          // lo fits, hi does not
    while (hi - lo > 1) {
        const int mid = lo + (hi - lo) / 2;
        if (!bytes(mid, &b)) return -1;
        (b <= budget ? lo : hi) = mid;
    }
    *n = lo;
    return 0;
}

size_t call_budget(t2v_vae* v, size_t cached) {
    if (v->budget != 0) return v->budget;
    size_t free_b = 0, total_b = 0;
    if (cudaMemGetInfo(&free_b, &total_b) != cudaSuccess) {
        cudaGetLastError();
        return SIZE_MAX;              // no reading: the whole-clip path, as before
    }
    const size_t avail = free_b + cached + v->gn_ws.bytes;
    return avail > kBudgetMargin ? avail - kBudgetMargin : 0;
}

// Runs a clip of `frames` frames through the plans of `cache`: as one plan if it is cached or fits the budget, else as
// ceil(frames / n) consecutive ranges of n frames (the last one the tail), n the largest that fits.  Before a plan is
// built, this direction's cached plans are dropped if the new one would not fit beside them.  A chunked call drops this
// direction's plans when it starts and again when it ends: its chunk plans are sized to the free memory, and keeping them
// would starve whatever runs next (the UNet after a vid2vid encode, a decode after it).  get(nf) returns the entry of an
// nf-frame plan (building it), run(entry, f0, nf) stages frames [f0, f0 + nf), replays the plan and writes the result.
template <class IO, class Get, class Run>
int run_in_chunks(t2v_vae* v, int dir, PlanCache<IO>& cache, const ParamStore& P, const char* what, int frames, int h, int w,
                  cudaStream_t stream, Get&& get, Run&& run) {
    int n = frames;
    size_t budget = SIZE_MAX;
    if (!cache.find(shape_key(frames, h, w), P.version())) {
        if (!P.complete(what)) return -1;
        budget = call_budget(v, cache.slab_bytes());
        size_t one = 0;
        const int rc = choose_chunk(v, dir, frames, h, w, budget, &n, &one);
        if (rc == -4) return rc;
        if (rc != 0) n = frames;      // dry pass failed: the build below reports why
    }
    const int n_chunks = (frames + n - 1) / n;
    const int tail = frames - (n_chunks - 1) * n;
    if (n_chunks > 1) cache.clear(stream);
    v->last_chunk[dir] = n;
    v->last_n_chunks[dir] = n_chunks;
    int rc = 0;
    for (int c = 0; c < n_chunks && rc == 0; ++c) {
        const int f0 = c * n, nf = c + 1 < n_chunks ? n : tail;
        if (budget != SIZE_MAX && !cache.find(shape_key(nf, h, w), P.version())) {
            size_t a = 0, g = 0;
            if (plan_bytes(v, dir, nf, h, w, &a, &g) == 0 && cache.slab_bytes() + a + g > budget) cache.clear(stream);
        }
        auto* e = get(nf);
        rc = e ? run(e, f0, nf) : -1;
    }
    if (n_chunks > 1) cache.clear(stream);
    return rc;
}

// A tap of the most recent decoder plan ("decoder.*") or encoder plan ("encoder.*"); null, with the error set, if none.
const std::pair<Tok, std::pair<int, int>>* find_tap(t2v_vae* v, const char* name) {
    auto* plan = strncmp(name, "encoder.", 8) == 0 ? (v->enc_plans.latest() ? v->enc_plans.latest()->plan.get() : nullptr)
                                                   : (v->plans.latest() ? v->plans.latest()->plan.get() : nullptr);
    if (plan) {
        auto it = plan->taps.find(name);
        if (it != plan->taps.end()) return &it->second;
    }
    set_error("VAE tap '%s' not found (enable taps before a whole-clip decode / encode)", name);
    return nullptr;
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
    int up = 1;
    for (int i = 1; i < v->cfg.n_mult; ++i) up *= 2;
    const long long pix = static_cast<long long>(h * up) * (w * up);      // pixels of one output frame
    const int zpad = (v->cfg.z_channels + 7) / 8 * 8;
    return run_in_chunks(
        v, DEC, v->plans, v->params, "VAE", frames, h, w, stream, [&](int nf) { return get_plan(v, nf, h, w, stream); },
        [&](PlanCache<VIO>::Entry* entry, int f0, int nf) {
            const VIO& io = entry->io;
            int rc = ingest_latent_frames(z, z_is_f32, io.z_tok, zpad, zpad, v->cfg.z_channels, F, h, w, f0, nf, z_scale, stream);
            if (rc != 0) return rc;
            rc = run_plan(entry->plan.get(), stream, true);
            if (rc != 0) {
                set_error("VAE launch failed (%d): %s", rc, cudaGetErrorString(cudaGetLastError()));
                return rc;
            }
            if (out_mode == 1)
                return frames_to_u8(io.out_tok, io.out_ld, reinterpret_cast<uint8_t*>(out) + f0 * pix * 3, nf * pix, stream);
            return frames_to_f32_nchw(io.out_tok, io.out_ld, reinterpret_cast<float*>(out) + f0 * pix * 3, nf, h * up, w * up, stream);
        });
}

int t2v_vae_encode(t2v_vae* v, const void* x, int x_is_f32, void* moments_out, int N, int H, int W, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    int down = 1;
    for (int i = 1; i < v->cfg.n_mult; ++i) down *= 2;
    if (N < 1 || H % down != 0 || W % down != 0) {
        set_error("t2v_vae_encode: H and W must be multiples of %d (got %d x %d)", down, H, W);
        return -3;
    }
    const long long in_frame = 3LL * H * W * (x_is_f32 ? 4 : 2);          // bytes of one input frame
    const int M = 2 * v->cfg.embed_dim;
    return run_in_chunks(
        v, ENC, v->enc_plans, v->enc_params, "VAE encoder", N, H, W, stream, [&](int nf) { return get_enc_plan(v, nf, H, W, stream); },
        [&](PlanCache<EncIO>::Entry* entry, int f0, int nf) {
            const EncIO& io = entry->io;
            int rc = ingest_latent(static_cast<const char*>(x) + f0 * in_frame, x_is_f32, io.x_tok, 8, 8, nf, 3, 1, H, W, 1.0f, stream);
            if (rc != 0) return rc;
            rc = run_plan(entry->plan.get(), stream, true);
            if (rc != 0) {
                set_error("VAE encoder launch failed (%d): %s", rc, cudaGetErrorString(cudaGetLastError()));
                return rc;
            }
            float* mom = static_cast<float*>(moments_out) + static_cast<long long>(f0) * M * io.ho * io.wo;
            return egress_latent(io.out_tok, io.out_ld, mom, 1, nf, M, 1, io.ho, io.wo, stream);
        });
}

double t2v_vae_flops(t2v_vae* v, int nframes, int h, int w) {
    VIO io;
    double flops = 0.0;
    if (dry_build(nullptr, false, [&](Plan* p, Arena* a, bool dry) { return build(v, p, a, dry, nullptr, nframes, h, w, &io); }, &flops) < 0)
        return -1.0;
    return flops;
}

int t2v_vae_plan_bytes(t2v_vae* v, int direction, int frames, int h, int w, size_t* arena, size_t* gn_workspace) {
    if (!v || !arena || !gn_workspace || (direction != DEC && direction != ENC) || frames < 1 || h < 1 || w < 1) return -1;
    if (plan_bytes(v, direction, frames, h, w, arena, gn_workspace) != 0) {
        set_error("t2v_vae_plan_bytes: the dry pass failed at %d frames of %d x %d", frames, h, w);
        return -1;
    }
    return 0;
}

int t2v_vae_plan_chunks(t2v_vae* v, int direction, int frames, int h, int w, size_t budget, int* chunk_frames, int* n_chunks) {
    if (!v || !chunk_frames || !n_chunks || (direction != DEC && direction != ENC) || frames < 1 || h < 1 || w < 1) return -1;
    int n = 0;
    size_t one = 0;
    const int rc = choose_chunk(v, direction, frames, h, w, budget, &n, &one);
    if (rc != 0) return rc;
    *chunk_frames = n;
    *n_chunks = (frames + n - 1) / n;
    return 0;
}

int t2v_vae_set_memory_budget(t2v_vae* v, size_t bytes) {
    if (!v) return -1;
    v->budget = bytes;
    return 0;
}

size_t t2v_vae_get_memory_budget(t2v_vae* v) { return v ? v->budget : 0; }

int t2v_vae_last_chunking(t2v_vae* v, int direction, int* chunk_frames, int* n_chunks) {
    if (!v || !chunk_frames || !n_chunks || (direction != DEC && direction != ENC)) return -1;
    *chunk_frames = v->last_chunk[direction];
    *n_chunks = v->last_n_chunks[direction];
    return 0;
}

int t2v_vae_cached_plans(t2v_vae* v, int direction, size_t* slab_bytes) {
    if (!v || (direction != DEC && direction != ENC)) return -1;
    const size_t n = direction == DEC ? v->plans.size() : v->enc_plans.size();
    if (slab_bytes) *slab_bytes = direction == DEC ? v->plans.slab_bytes() : v->enc_plans.slab_bytes();
    return static_cast<int>(n);
}

int t2v_vae_enable_taps(t2v_vae* v, int on, void* stream) {
    if (!v) return -1;
    v->taps_enabled = on != 0;
    v->plans.clear(reinterpret_cast<cudaStream_t>(stream));
    v->enc_plans.clear(reinterpret_cast<cudaStream_t>(stream));
    return 0;
}

int t2v_vae_tap_info(t2v_vae* v, const char* name, long long* rows, int* C, int* h, int* w) {
    const auto* tap = find_tap(v, name);
    if (!tap) return -1;
    if (rows) *rows = tap->first.rows;
    if (C) *C = tap->first.C;
    if (h) *h = tap->second.first;
    if (w) *w = tap->second.second;
    return 0;
}

long long t2v_vae_read_tap(t2v_vae* v, const char* name, void* dst, long long cap_elems, void* stream_) {
    const auto* tap = find_tap(v, name);
    if (!tap) return -1;
    const Tok& t = tap->first;
    const int h = tap->second.first, w = tap->second.second;
    const long long n = t.rows * t.C;
    if (n > cap_elems) {
        set_error("VAE tap '%s' needs %lld elements", name, n);
        return -2;
    }
    // [frames, h, w, C] tokens -> fp16 [frames, C, h, w]
    const int frames = static_cast<int>(t.rows / (static_cast<long long>(h) * w));
    if (egress_latent(t.p, t.ld, dst, 0, frames, t.C, 1, h, w, reinterpret_cast<cudaStream_t>(stream_)) != 0) return -3;
    return n;
}

}  // extern "C"
