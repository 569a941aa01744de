// VideoCrafter's T2I-Adapter (videocrafter/lvdm/models/modules/adapter.py: Adapter, ResnetBlock, Downsample) as a
// pre-planned launch list: the depth-conditioning network that T2VAdapterDepth.get_adapter_features runs once per clip
// (videocrafter/lvdm/models/ddpm3d.py:1470-1484), every frame of the clip in one batch.
//
//   x = conv_in(PixelUnshuffle(8)(cond))                                  3x3, cin -> channels[0]
//   for level i, block j:   (k = i * nums_rb + j)
//       x = down_opt(x)          if i > 0 and j == 0: 3x3 stride-2 pad-1 conv (use_conv) or 2x2 average pooling
//       x = in_conv(x)           if in_c != out_c or not sk (ksize x ksize)
//       x = block2(relu(block1(x))) + (skep(x) if not sk else x)          block1 3x3, block2 / skep ksize x ksize
//   one feature map per level: x after the level's last block
//
// Same engine as the denoiser: channels-last tokens [(n, y, x), C] fp16, every conv on the wgmma implicit GEMM (3x3: nine
// taps over the frame grid, 1x1: a plain linear, stride 2: the stride-2 gather + one GEMM).  The residual add is the
// epilogue of block2's GEMM (sk) or of skep's GEMM with block2's output as its residual operand (not sk).  PixelUnshuffle,
// the ReLU and the average pooling are small kernels in elementwise.cu.
#include "../../include/t2v_b200.h"
#include "runtime.cuh"

#include <cstdio>
#include <cstring>
#include <memory>

using namespace t2v;

namespace t2v {
namespace {

struct AdapterIO {
    __half* cond_tok = nullptr;          // PixelUnshuffle'd input [N*(H/8)*(W/8), cin]
    __half* feat[4] = {nullptr, nullptr, nullptr, nullptr};
    long long feat_elems[4] = {0, 0, 0, 0};
};

}  // namespace
}  // namespace t2v

struct t2v_adapter {
    t2v_adapter_config cfg;
    ParamStore params;
    PlanCache<AdapterIO> plans{4};      // key: "N,H,W"
};

namespace t2v {
namespace {

std::string body(int k) { return "body." + std::to_string(k); }

bool has_in_conv(const t2v_adapter_config& c, int in_c, int out_c) { return in_c != out_c || !c.sk; }

void expect_params(t2v_adapter* a) {
    ParamStore& P = a->params;
    const t2v_adapter_config& c = a->cfg;
    auto conv = [&](const std::string& p, int o, int i, int k) {
        P.expect(p + ".weight", {o, i, k, k});
        P.expect(p + ".bias", {o});
    };
    conv("conv_in", c.channels[0], c.cin, 3);
    for (int i = 0; i < c.n_levels; ++i)
        for (int j = 0; j < c.nums_rb; ++j) {
            const std::string p = body(i * c.nums_rb + j);
            const bool down = i > 0 && j == 0;
            const int in_c = down ? c.channels[i - 1] : c.channels[i], out_c = c.channels[i];
            if (has_in_conv(c, in_c, out_c)) conv(p + ".in_conv", out_c, in_c, c.ksize);
            conv(p + ".block1", out_c, out_c, 3);
            conv(p + ".block2", out_c, out_c, c.ksize);
            if (!c.sk) conv(p + ".skep", out_c, in_c, c.ksize);
            if (down && c.use_conv) conv(p + ".down_opt.op", in_c, in_c, 3);
        }
}

// Conv2d(k, stride 1, padding k // 2) for k in {1, 3}, bias, optional residual in the epilogue
Tok conv_k(NetCtx& c, const Tok& x, const std::string& p, int k, int N, int hc, int wc, const Tok* residual) {
    if (k == 3) return conv3x3(c, x, p + ".weight", prm(c, p + ".bias"), 0, 0, N, hc, wc, residual);
    return linear(c, x, w_conv(c, p + ".weight", 1), N, prm(c, p + ".bias"), residual);
}

// level sizes: PixelUnshuffle(8), then every level after the first halves them (conv: rounding up, pooling: down)
void level_sizes(const t2v_adapter_config& c, int H, int W, int* hs, int* ws) {
    int h = H / 8, w = W / 8;
    for (int i = 0; i < c.n_levels; ++i) {
        if (i > 0) {
            h = c.use_conv ? (h + 1) / 2 : h / 2;
            w = c.use_conv ? (w + 1) / 2 : w / 2;
        }
        hs[i] = h;
        ws[i] = w;
    }
}

int build(t2v_adapter* a, Plan* plan, Arena* arena, bool dry, cudaStream_t stream, int N, int H, int W, AdapterIO* io) {
    Builder bld(plan, arena, dry, num_sms());
    NetCtx c{&a->params, &bld, stream, nullptr};
    const t2v_adapter_config& cfg = a->cfg;
    int hc = H / 8, wc = W / 8;
    const long long R0 = static_cast<long long>(N) * hc * wc;
    Tok x0 = bld.alloc(R0, cfg.cin);
    io->cond_tok = x0.p;
    Tok x = conv3x3(c, x0, "conv_in.weight", prm(c, "conv_in.bias"), 0, 0, cfg.channels[0], hc, wc, nullptr);
    bld.free(x0);
    // a finished level's feature map stays live (it is copied out after the launch list); everything else is released
    int done = 0;
    auto release = [&](const Tok& t) {
        for (int l = 0; l < done; ++l)
            if (io->feat[l] == t.p) return;
        bld.free(t);
    };
    for (int i = 0; i < cfg.n_levels; ++i) {
        for (int j = 0; j < cfg.nums_rb; ++j) {
            const std::string p = body(i * cfg.nums_rb + j);
            const bool down = i > 0 && j == 0;
            const int in_c = down ? cfg.channels[i - 1] : cfg.channels[i], out_c = cfg.channels[i];
            if (down) {
                Tok y;
                if (cfg.use_conv) {            // Conv2d(in_c, in_c, 3, stride 2, padding 1): output (h + 1) / 2
                    const int ho = (hc + 1) / 2, wo = (wc + 1) / 2;
                    Tok col = bld.alloc(static_cast<long long>(N) * ho * wo, 9 * in_c);
                    const Tok xx = x;
                    const int hh = hc, ww = wc;
                    bld.step([=](cudaStream_t s) { return im2col_s2(xx.p, col.p, N, hh, ww, xx.C, s); }, 1, STEP_OTHER, 0.0,
                             "adapter stride-2 gather");
                    y = linear(c, col, w_conv_kmajor(c, p + ".down_opt.op.weight"), in_c, prm(c, p + ".down_opt.op.bias"), nullptr);
                    bld.free(col);
                    hc = ho;
                    wc = wo;
                } else {                       // AvgPool2d(2, 2): output h / 2
                    const int ho = hc / 2, wo = wc / 2;
                    y = bld.alloc(static_cast<long long>(N) * ho * wo, in_c);
                    const Tok xx = x;
                    const int hh = hc, ww = wc;
                    bld.step([=](cudaStream_t s) { return avgpool2x2(xx.p, y.p, N, hh, ww, xx.C, s); }, 1, STEP_OTHER, 0.0,
                             "adapter avgpool 2x2");
                    hc = ho;
                    wc = wo;
                }
                release(x);
                x = y;
            }
            if (has_in_conv(cfg, in_c, out_c)) {
                Tok y = conv_k(c, x, p + ".in_conv", cfg.ksize, out_c, hc, wc, nullptr);
                release(x);
                x = y;
            }
            Tok h = conv3x3(c, x, p + ".block1.weight", prm(c, p + ".block1.bias"), 0, 0, out_c, hc, wc, nullptr);
            {
                const Tok hh = h;
                bld.step([=](cudaStream_t s) { return relu_inplace(hh.p, hh.rows, hh.C, s); }, 1, STEP_OTHER, 0.0, "adapter relu");
            }
            Tok y;
            if (cfg.sk) {                      // h + x in block2's epilogue
                y = conv_k(c, h, p + ".block2", cfg.ksize, out_c, hc, wc, &x);
                bld.free(h);
            } else {                           // block2(h) as the residual operand of skep's GEMM: skep(x) + block2(h)
                Tok h2 = conv_k(c, h, p + ".block2", cfg.ksize, out_c, hc, wc, nullptr);
                bld.free(h);
                y = conv_k(c, x, p + ".skep", cfg.ksize, out_c, hc, wc, &h2);
                bld.free(h2);
            }
            release(x);
            x = y;
        }
        io->feat[i] = x.p;
        io->feat_elems[i] = x.rows * x.C;
        done = i + 1;
    }
    return bld.error;
}

PlanCache<AdapterIO>::Entry* get_plan(t2v_adapter* a, int N, int H, int W, cudaStream_t stream) {
    const std::string key = std::to_string(N) + "," + std::to_string(H) + "," + std::to_string(W);
    if (auto* e = a->plans.find(key, a->params.version())) return e;
    if (!a->params.complete("Adapter")) return nullptr;
    return a->plans.build(key, a->params.version(), stream, std::unique_ptr<Plan>(new Plan()), false, "Adapter",
                          [&](Plan* p, Arena* ar, bool dry, AdapterIO* io) { return build(a, p, ar, dry, stream, N, H, W, io); });
}

}  // namespace
}  // namespace t2v

extern "C" {

int t2v_adapter_create(const t2v_adapter_config* cfg, t2v_adapter** out) {
    if (!cfg || !out) return -1;
    if (cfg->n_levels < 1 || cfg->n_levels > 4 || cfg->nums_rb < 1) {
        set_error("Adapter: 1 to 4 levels (got %d) and nums_rb >= 1 (got %d)", cfg->n_levels, cfg->nums_rb);
        return -2;
    }
    if (cfg->cin < 64 || cfg->cin % 64 != 0) {
        set_error("Adapter: cin must be a multiple of 64 (PixelUnshuffle(8) of cin / 64 condition channels; got %d)", cfg->cin);
        return -2;
    }
    if (cfg->ksize != 1 && cfg->ksize != 3) {
        set_error("Adapter: ksize %d is not built (1 or 3)", cfg->ksize);
        return -2;
    }
    for (int i = 0; i < cfg->n_levels; ++i)
        if (cfg->channels[i] < 8 || cfg->channels[i] % 8 != 0) {
            set_error("Adapter: every level width must be a positive multiple of 8 (channels[%d] = %d)", i, cfg->channels[i]);
            return -2;
        }
    if (!cfg->sk)        // the reference builds skep for in_c channels but applies it after in_conv (out_c channels)
        for (int i = 1; i < cfg->n_levels; ++i)
            if (cfg->channels[i] != cfg->channels[i - 1]) {
                set_error("Adapter: sk=False with differing level widths (%d -> %d) cannot run: the reference applies skep, "
                          "built for the block's input width, to in_conv's output", cfg->channels[i - 1], cfg->channels[i]);
                return -2;
            }
    t2v_adapter* a = new t2v_adapter();
    a->cfg = *cfg;
    expect_params(a);
    *out = a;
    return 0;
}

void t2v_adapter_destroy(t2v_adapter* a) { delete a; }

int t2v_adapter_set_param(t2v_adapter* a, const char* name, const void* data, int dtype, int ndim, const int64_t* shape,
                          void* stream) {
    return a->params.set(name, data, dtype, ndim, shape, reinterpret_cast<cudaStream_t>(stream));
}

int t2v_adapter_missing_params(t2v_adapter* a, char* name_out, size_t name_cap) {
    return missing_params_out(a->params, name_out, name_cap);
}

int t2v_adapter_param_info(t2v_adapter* a, int index, char* name_out, size_t name_cap, int64_t* shape_out, int* ndim_out) {
    return param_info_out(a->params, index, name_out, name_cap, shape_out, ndim_out);
}

int t2v_adapter_lora_apply(t2v_adapter* a, const char* weight_name, const void* up, const void* down, int dtype, int rank, float alpha,
                           void* stream) {
    clear_pending_error("t2v_adapter_lora_apply");
    return a->params.lora_apply(weight_name, up, down, dtype, rank, alpha, reinterpret_cast<cudaStream_t>(stream));
}

int t2v_adapter_lora_restore(t2v_adapter* a, const char* weight_name, void* stream) {
    clear_pending_error("t2v_adapter_lora_restore");
    return a->params.lora_restore(weight_name, reinterpret_cast<cudaStream_t>(stream));
}

int t2v_adapter_lora_clear(t2v_adapter* a, void* stream) { return a->params.lora_clear(reinterpret_cast<cudaStream_t>(stream)); }

int t2v_adapter_lora_merged(t2v_adapter* a) { return a->params.merged_count(); }

int t2v_adapter_encode(t2v_adapter* a, const void* cond, int cond_is_f32, void* const* feats_out, int N, int H, int W,
                       void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    clear_pending_error("t2v_adapter_encode");
    const t2v_adapter_config& cfg = a->cfg;
    if (N < 1 || H < 8 || W < 8 || H % 8 != 0 || W % 8 != 0) {
        set_error("Adapter: condition frames must be at least 8x8 with H and W multiples of 8 (PixelUnshuffle(8)); got %d frames "
                  "of %dx%d", N, H, W);
        return -2;
    }
    int hs[4], ws[4];
    level_sizes(cfg, H, W, hs, ws);
    for (int i = 0; i < cfg.n_levels; ++i)
        if (hs[i] < 1 || ws[i] < 1) {
            set_error("Adapter: level %d of a %dx%d input would be empty (%dx%d after %s)", i, H, W, hs[i], ws[i],
                      cfg.use_conv ? "stride-2 convs" : "2x2 average pooling");
            return -3;
        }
    auto* entry = get_plan(a, N, H, W, stream);
    if (!entry) return -1;
    const AdapterIO& io = entry->io;
    int rc = pixel_unshuffle_ingest(cond, cond_is_f32, io.cond_tok, N, cfg.cin / 64, H, W, stream);
    if (rc != 0) return rc;
    rc = run_plan(entry->plan.get(), stream, true);
    if (rc != 0) {
        set_error("Adapter launch failed (%d): %s", rc, cudaGetErrorString(cudaGetLastError()));
        return rc;
    }
    for (int i = 0; i < cfg.n_levels; ++i)
        if (cudaMemcpyAsync(feats_out[i], io.feat[i], static_cast<size_t>(io.feat_elems[i]) * sizeof(__half), cudaMemcpyDeviceToDevice,
                            stream) != cudaSuccess)
            return launch_status("adapter feature copy");
    return launch_status("adapter launch");
}

}  // extern "C"
