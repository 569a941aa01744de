// ModelScope UNetSD denoiser as a pre-planned launch list (replaces modelscope/t2v_model.py:98-501).
//
// One activation layout for the whole network: channels-last tokens  X[(b, f, y, x), C]  fp16.
//   * spatial modules (ResBlock convs, SpatialTransformer, Down/Upsample) see rows grouped per frame,
//   * temporal modules (TemporalConvBlock_v2, TemporalTransformer) address the SAME buffer with a frame stride,
// so none of the reference's `(b f) c h w <-> b c f h w <-> (b h w) f c` rearrange copies exist here.
// Every contraction goes through the wgmma implicit-GEMM engine (gemm_tc.cu); norms / attention / glue are the
// kernels in norm.cu, attention.cu, elementwise.cu.
#include "../../include/t2v_b200.h"
#include "runtime.cuh"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <memory>

namespace t2v {

namespace {

struct Blk {
    enum Kind { STEM, RES, ST, TT, DOWN, UP, STT } kind;     // STT: VideoCrafter SpatialTemporalTransformer
    std::string prefix;
    int cin = 0, cout = 0, heads = 0, inner = 0;
};

constexpr int kMaxFeat = 8;

struct IO {
    __half* x_tok;      // [R, 8]
    float* t;           // [B]
    __half* ctx;        // [Bc*L, context_dim]
    __half* out_tok;    // [R, 8]
    // adapter features (plans built with feats_B > 0): staging [feats_B * F * h_i * w_i, C_i] per injection point
    int n_feat = 0;
    __half* feat[kMaxFeat] = {nullptr};
    long long feat_elems[kMaxFeat] = {0};
};

int max_plans() {
    static const int n = getenv("T2V_MAX_PLANS") ? std::max(1, atoi(getenv("T2V_MAX_PLANS"))) : 4;
    return n;
}

}  // namespace

}  // namespace t2v

using namespace t2v;

struct t2v_unet {
    t2v_unet_config cfg;
    ParamStore params;
    std::vector<std::vector<Blk>> ins, outs;
    std::vector<Blk> mid;
    PlanCache<IO> plans{max_plans()};                        // key: plan_key()
    bool taps_enabled = false;
    int last_launches = 0;
    int last_exchanges = 0;
    GnWorkspace gn_ws;
    // frame-sharded clip (shard.cuh): one rank of `peers.nranks`, comm = this rank's IPC-shared flag / GroupNorm region
    bool shard_on = false;
    ShardPeers peers;
    ShardComm* comm = nullptr;
    t2v_unet() { memset(&peers, 0, sizeof(peers)); }
    ~t2v_unet() {
        plans.clear(nullptr);               // closes the peers' slab mappings before the comm mappings go
        for (int r = 0; r < SHARD_MAX_RANKS; ++r)
            if (peers.comm[r] != nullptr && peers.comm[r] != comm) cudaIpcCloseMemHandle(peers.comm[r]);
        if (comm) cudaFree(comm);
    }
};

namespace t2v {
namespace {

bool in_scales(const t2v_unet_config& c, float s) {
    for (int i = 0; i < c.n_attn_scales; ++i)
        if (std::fabs(c.attn_scales[i] - s) < 1e-9f) return true;
    return false;
}

// mirrors UNetSD.__init__ (t2v_model.py:148-323): which modules exist, with which channel counts and names
void enumerate(t2v_unet* u) {
    const t2v_unet_config& c = u->cfg;
    const int dim = c.dim, hd = c.head_dim, nm = c.n_mult;
    std::vector<int> enc, dec, shortcut;
    enc.push_back(dim);
    for (int i = 0; i < nm; ++i) enc.push_back(dim * c.dim_mult[i]);
    dec.push_back(dim * c.dim_mult[nm - 1]);
    for (int i = nm - 1; i >= 0; --i) dec.push_back(dim * c.dim_mult[i]);
    float scale = 1.0f;
    auto name = [](const char* base, int n, int k) {
        char buf[64];
        snprintf(buf, sizeof(buf), "%s.%d.%d", base, n, k);
        return std::string(buf);
    };
    u->ins.push_back({Blk{Blk::STEM, "input_blocks.0.0", c.in_dim, dim, 0, 0},
                      Blk{Blk::TT, "input_blocks.0.1", dim, dim, c.num_heads, c.num_heads * hd}});
    shortcut.push_back(dim);
    for (int i = 0; i < nm; ++i) {
        int cin = enc[i];
        const int cout = enc[i + 1];
        for (int j = 0; j < c.num_res_blocks; ++j) {
            const int n = static_cast<int>(u->ins.size());
            std::vector<Blk> blk;
            blk.push_back(Blk{Blk::RES, name("input_blocks", n, 0), cin, cout, 0, 0});
            if (in_scales(c, scale)) {
                blk.push_back(Blk{Blk::ST, name("input_blocks", n, 1), cout, cout, cout / hd, cout});
                blk.push_back(Blk{Blk::TT, name("input_blocks", n, 2), cout, cout, cout / hd, cout});
            }
            cin = cout;
            u->ins.push_back(blk);
            shortcut.push_back(cout);
            if (i != nm - 1 && j == c.num_res_blocks - 1) {
                char buf[64];
                snprintf(buf, sizeof(buf), "input_blocks.%d", static_cast<int>(u->ins.size()));
                u->ins.push_back({Blk{Blk::DOWN, buf, cout, cout, 0, 0}});
                shortcut.push_back(cout);
                scale /= 2.0f;
            }
        }
    }
    const int cm = enc.back();
    u->mid = {Blk{Blk::RES, "middle_block.0", cm, cm, 0, 0}, Blk{Blk::ST, "middle_block.1", cm, cm, cm / hd, cm},
              Blk{Blk::TT, "middle_block.2", cm, cm, cm / hd, cm}, Blk{Blk::RES, "middle_block.3", cm, cm, 0, 0}};
    for (int i = 0; i < nm; ++i) {
        int cin = dec[i];
        const int cout = dec[i + 1];
        for (int j = 0; j < c.num_res_blocks + 1; ++j) {
            const int n = static_cast<int>(u->outs.size());
            std::vector<Blk> blk;
            blk.push_back(Blk{Blk::RES, name("output_blocks", n, 0), cin + shortcut.back(), cout, 0, 0});
            shortcut.pop_back();
            int k = 1;
            if (in_scales(c, scale)) {
                blk.push_back(Blk{Blk::ST, name("output_blocks", n, 1), cout, cout, cout / hd, cout});
                blk.push_back(Blk{Blk::TT, name("output_blocks", n, 2), cout, cout, cout / hd, cout});
                k = 3;
            }
            cin = cout;
            if (i != nm - 1 && j == c.num_res_blocks) {
                blk.push_back(Blk{Blk::UP, name("output_blocks", n, k), cout, cout, 0, 0});
                scale *= 2.0f;
            }
            u->outs.push_back(blk);
        }
    }
}

void expect_params(t2v_unet* u) {
    ParamStore& P = u->params;
    const t2v_unet_config& c = u->cfg;
    const int E = c.dim * 4;
    auto lin = [&](const std::string& p, int o, int i, bool bias = true) {
        P.expect(p + ".weight", {o, i});
        if (bias) P.expect(p + ".bias", {o});
    };
    auto norm = [&](const std::string& p, int ch) {
        P.expect(p + ".weight", {ch});
        P.expect(p + ".bias", {ch});
    };
    auto tblock = [&](const std::string& p, int inner, int ctx) {
        for (int a = 0; a < 2; ++a) {
            const std::string ap = p + (a == 0 ? ".attn1" : ".attn2");
            const int cd = a == 0 ? inner : ctx;
            lin(ap + ".to_q", inner, inner, false);
            lin(ap + ".to_k", inner, cd, false);
            lin(ap + ".to_v", inner, cd, false);
            lin(ap + ".to_out.0", inner, inner);
        }
        lin(p + ".ff.net.0.proj", inner * 8, inner);
        lin(p + ".ff.net.2", inner, inner * 4);
        norm(p + ".norm1", inner);
        norm(p + ".norm2", inner);
        norm(p + ".norm3", inner);
    };
    lin("time_embed.0", E, c.dim);
    lin("time_embed.2", E, E);
    std::vector<Blk> all;
    for (auto& b : u->ins) all.insert(all.end(), b.begin(), b.end());
    all.insert(all.end(), u->mid.begin(), u->mid.end());
    for (auto& b : u->outs) all.insert(all.end(), b.begin(), b.end());
    for (const Blk& b : all) {
        const std::string& p = b.prefix;
        switch (b.kind) {
            case Blk::STEM:
                P.expect(p + ".weight", {b.cout, b.cin, 3, 3});
                P.expect(p + ".bias", {b.cout});
                break;
            case Blk::RES: {
                norm(p + ".in_layers.0", b.cin);
                P.expect(p + ".in_layers.2.weight", {b.cout, b.cin, 3, 3});
                P.expect(p + ".in_layers.2.bias", {b.cout});
                lin(p + ".emb_layers.1", b.cout, E);
                norm(p + ".out_layers.0", b.cout);
                P.expect(p + ".out_layers.3.weight", {b.cout, b.cout, 3, 3});
                P.expect(p + ".out_layers.3.bias", {b.cout});
                if (b.cin != b.cout) {
                    P.expect(p + ".skip_connection.weight", {b.cout, b.cin, 1, 1});
                    P.expect(p + ".skip_connection.bias", {b.cout});
                }
                const char* names[4] = {"conv1", "conv2", "conv3", "conv4"};
                const int idx[4] = {2, 3, 3, 3};     // conv1 has no Dropout slot (t2v_model.py:1201-1212)
                for (int i = 0; i < 4; ++i) {
                    const std::string tp = p + ".temopral_conv." + names[i];   // sic: checkpoint key (t2v_model.py:968)
                    norm(tp + ".0", b.cout);
                    P.expect(tp + "." + std::to_string(idx[i]) + ".weight", {b.cout, b.cout, 3, 1, 1});
                    P.expect(tp + "." + std::to_string(idx[i]) + ".bias", {b.cout});
                }
                break;
            }
            case Blk::ST:
                norm(p + ".norm", b.cin);
                lin(p + ".proj_in", b.inner, b.cin);
                tblock(p + ".transformer_blocks.0", b.inner, c.context_dim);
                lin(p + ".proj_out", b.cin, b.inner);
                break;
            case Blk::TT:
                norm(p + ".norm", b.cin);
                P.expect(p + ".proj_in.weight", {b.inner, b.cin, 1});
                P.expect(p + ".proj_in.bias", {b.inner});
                tblock(p + ".transformer_blocks.0", b.inner, b.inner);
                P.expect(p + ".proj_out.weight", {b.cin, b.inner, 1});
                P.expect(p + ".proj_out.bias", {b.cin});
                break;
            case Blk::DOWN:
                P.expect(p + ".op.weight", {b.cout, b.cin, 3, 3});
                P.expect(p + ".op.bias", {b.cout});
                break;
            case Blk::UP:
                P.expect(p + ".conv.weight", {b.cout, b.cin, 3, 3});
                P.expect(p + ".conv.bias", {b.cout});
                break;
        }
    }
    norm("out.0", c.dim);
    P.expect("out.2.weight", {c.out_dim, c.dim, 3, 3});
    P.expect("out.2.bias", {c.out_dim});
}


// ---- VideoCrafter (arch 1): mirrors UNetModel.__init__ (videocrafter/lvdm/models/modules/openaimodel3d.py:407-617) with
// legacy = False, num_head_channels = -1 (dim_head = ch / num_heads), resblock_updown = False, kernel_size_t = 1
void enumerate_vc(t2v_unet* u) {
    const t2v_unet_config& c = u->cfg;
    const int mc = c.dim, nm = c.n_mult;
    auto name = [](const char* base, int n, int k) {
        char buf[64];
        snprintf(buf, sizeof(buf), "%s.%d.%d", base, n, k);
        return std::string(buf);
    };
    u->ins.push_back({Blk{Blk::STEM, "input_blocks.0.0", c.in_dim, mc, 0, 0}});
    std::vector<int> chans{mc};
    int ch = mc;
    float scale = 1.0f;
    for (int level = 0; level < nm; ++level) {
        for (int j = 0; j < c.num_res_blocks; ++j) {
            const int n = static_cast<int>(u->ins.size());
            std::vector<Blk> blk;
            blk.push_back(Blk{Blk::RES, name("input_blocks", n, 0), ch, mc * c.dim_mult[level], 0, 0});
            ch = mc * c.dim_mult[level];
            if (in_scales(c, scale)) blk.push_back(Blk{Blk::STT, name("input_blocks", n, 1), ch, ch, c.num_heads, ch});
            u->ins.push_back(blk);
            chans.push_back(ch);
        }
        if (level != nm - 1) {
            const int n = static_cast<int>(u->ins.size());
            u->ins.push_back({Blk{Blk::DOWN, name("input_blocks", n, 0), ch, ch, 0, 0}});
            chans.push_back(ch);
            scale /= 2.0f;
        }
    }
    u->mid = {Blk{Blk::RES, "middle_block.0", ch, ch, 0, 0}, Blk{Blk::STT, "middle_block.1", ch, ch, c.num_heads, ch},
              Blk{Blk::RES, "middle_block.2", ch, ch, 0, 0}};
    for (int level = nm - 1; level >= 0; --level) {
        for (int i = 0; i < c.num_res_blocks + 1; ++i) {
            const int n = static_cast<int>(u->outs.size());
            const int ich = chans.back();
            chans.pop_back();
            std::vector<Blk> blk;
            blk.push_back(Blk{Blk::RES, name("output_blocks", n, 0), ch + ich, mc * c.dim_mult[level], 0, 0});
            ch = mc * c.dim_mult[level];
            if (in_scales(c, scale))
                blk.push_back(Blk{Blk::STT, name("output_blocks", n, static_cast<int>(blk.size())), ch, ch, c.num_heads, ch});
            if (level != 0 && i == c.num_res_blocks) {
                blk.push_back(Blk{Blk::UP, name("output_blocks", n, static_cast<int>(blk.size())), ch, ch, 0, 0});
                scale *= 2.0f;
            }
            u->outs.push_back(blk);
        }
    }
}

void expect_params_vc(t2v_unet* u) {
    ParamStore& P = u->params;
    const t2v_unet_config& c = u->cfg;
    const int E = c.dim * 4;
    auto lin = [&](const std::string& p, int o, int i, bool bias = true) {
        P.expect(p + ".weight", {o, i});
        if (bias) P.expect(p + ".bias", {o});
    };
    auto norm = [&](const std::string& p, int ch) {
        P.expect(p + ".weight", {ch});
        P.expect(p + ".bias", {ch});
    };
    auto conv = [&](const std::string& p, int o, int i, int k) {
        P.expect(p + ".weight", {o, i, 1, k, k});
        P.expect(p + ".bias", {o});
    };
    lin("time_embed.0", E, c.dim);
    lin("time_embed.2", E, E);
    std::vector<Blk> all;
    for (auto& b : u->ins) all.insert(all.end(), b.begin(), b.end());
    all.insert(all.end(), u->mid.begin(), u->mid.end());
    for (auto& b : u->outs) all.insert(all.end(), b.begin(), b.end());
    for (const Blk& b : all) {
        const std::string& p = b.prefix;
        switch (b.kind) {
            case Blk::STEM: conv(p, b.cout, b.cin, 3); break;
            case Blk::RES:
                norm(p + ".in_layers.0", b.cin);
                conv(p + ".in_layers.2", b.cout, b.cin, 3);
                lin(p + ".emb_layers.1", b.cout, E);
                norm(p + ".out_layers.0", b.cout);
                conv(p + ".out_layers.3", b.cout, b.cout, 3);
                if (b.cin != b.cout) conv(p + ".skip_connection", b.cout, b.cin, 1);
                break;
            case Blk::STT: {
                const int inner = b.inner, d = inner / b.heads;
                norm(p + ".norm", b.cin);
                conv(p + ".proj_in", inner, b.cin, 1);
                conv(p + ".proj_out", b.cin, inner, 1);
                const std::string t = p + ".transformer_blocks.0";
                const char* att[4] = {"attn1", "attn2", "attn1_tmp", "attn2_tmp"};
                for (int a = 0; a < 4; ++a) {
                    const std::string ap = t + "." + att[a];
                    const int kd = a == 1 ? c.context_dim : inner;
                    lin(ap + ".to_q", inner, inner, false);
                    lin(ap + ".to_k", inner, kd, false);
                    lin(ap + ".to_v", inner, kd, false);
                    lin(ap + ".to_out.0", inner, inner);
                    if (a >= 2) {
                        P.expect(ap + ".relative_position_k.embeddings_table", {2 * c.temporal_length + 1, d});
                        P.expect(ap + ".relative_position_v.embeddings_table", {2 * c.temporal_length + 1, d});
                    }
                }
                lin(t + ".ff.net.0.proj", inner * 8, inner);
                lin(t + ".ff.net.2", inner, inner * 4);
                for (int n = 1; n <= 5; ++n) norm(t + ".norm" + std::to_string(n), inner);
                break;
            }
            case Blk::DOWN: conv(p + ".op", b.cout, b.cin, 3); break;
            case Blk::UP: conv(p + ".conv", b.cout, b.cin, 3); break;
            default: break;
        }
    }
    norm("out.0", c.dim);
    conv("out.2", c.out_dim, c.dim, 3);
}

// ------------------------------------------------------------------------------------------ plan construction
struct Ctx : NetCtx {
    t2v_unet* u;
    int B, F, h, w, L;
    int Bc;                   // context batch: sample j reads prompt j / (B / Bc); = B when every sample brings its own
    int Fl;                   // frames held by this rank in the frame-sharded (FS) layout; = F when the clip is not sharded
    int rank, nranks;         // (0, 1) when not sharded
    char* slab;               // base of the plan's activation slab (exchange destinations are published as offsets into it)
    __half* emb;              // [B, E] time embedding (after time_embed MLP)
    __half* ctx;              // [Bc*L, ctx_dim] fixed staging of the text conditioning
    Plan* plan;
};

// pixels of a (hcur x wcur) level this rank owns in the pixel-sharded (PS) layout
int own_pixels(const Ctx& c, int hcur, int wcur) {
    if (c.nranks <= 1) return hcur * wcur;
    int pb[SHARD_MAX_RANKS + 1];
    shard_partition(hcur * wcur, c.nranks, pb);
    return pb[c.rank + 1] - pb[c.rank];
}

// FS <-> PS transpose of a sharded clip's token matrix (shard.cu): every rank pushes its blocks into the peers' buffers
Tok exchange(Ctx& c, const Tok& x, bool to_ps, int hcur, int wcur) {
    const int P = hcur * wcur;
    const int np = own_pixels(c, hcur, wcur);
    const long long rows = to_ps ? static_cast<long long>(c.B) * c.F * np : static_cast<long long>(c.B) * c.Fl * P;
    Tok y = c.b->alloc(rows, x.C);
    PlanShard* ps = c.plan_shard;
    const int k = ps->n_xchg++;
    if (k >= SHARD_MAX_XCHG - 1) {          // the last slot is the barrier's
        set_error("frame-sharded plan: more than %d layout exchanges", SHARD_MAX_XCHG - 1);
        c.b->error = -31;
        return y;
    }
    if (!c.b->dry()) ps->dst_off[k] = reinterpret_cast<char*>(y.p) - c.slab;
    XchgParams xp;
    memset(&xp, 0, sizeof(xp));
    xp.slot = k;
    xp.to_ps = to_ps ? 1 : 0;
    xp.B = c.B; xp.F = c.F; xp.P = P; xp.C = x.C;
    xp.ld_src = x.ld; xp.ld_dst = y.ld;
    xp.src = x.p;
    for (int r = 0; r <= c.nranks; ++r) xp.fb[r] = ps->fb[r];
    shard_partition(P, c.nranks, xp.pb);
    const ShardPeers* peers = c.shard_peers;
    const int me = c.rank, nr = c.nranks, sms = c.b->sms();
    __half* own = y.p;
    char lab[96];
    snprintf(lab, sizeof(lab), "exchange %s rows=%lld C=%d", to_ps ? "FS->PS" : "PS->FS", rows, x.C);
    c.b->step([=](cudaStream_t s) {
        if (!ps->connected) return -40;         // t2v_unet_shard_connect has not run for this plan
        XchgParams q = xp;
        q.peers = *peers;
        for (int r = 0; r < nr; ++r)
            q.dst[r] = r == me ? own : reinterpret_cast<__half*>(ps->peer_slab[r] + ps->peer_dst_off[r][k]);
        return shard_exchange(q, sms, s);
    }, 1, STEP_OTHER, 0.0, lab);
    return y;
}

void tap(Ctx& c, const std::string& name, const Tok& t, int h, int w) {
    if (c.u->taps_enabled && !c.b->dry()) c.plan->taps[name] = {t, {h, w}};
}

// GroupNorm rows per instance of a spatial module over P pixels per frame: ModelScope normalises each frame on its own
// (4-D input), VideoCrafter's GroupNorm32 takes a sample's statistics over all its frames (5-D input, util.py:271-273)
long long norm_rows(const Ctx& c, long long P) { return c.u->cfg.arch == 1 ? P * c.F : P; }

// ---- transformer sub-layers of ModelScope's BasicTransformerBlock (t2v_model.py:803-809) and VideoCrafter's
// BasicTransformerBlockST (attention_temporal.py:301-335): x + to_out(attention(LN x)) and x + FF(LN x), every LayerNorm
// folded into the GEMM that consumes it.  Each frees what it consumed, x included, and returns the new x.
// Heads of width d = C / heads, scale d^-0.5 (0.125 at ModelScope's d = 64).

AttnParams attn_params(const Tok& o, int heads) {
    AttnParams a;
    memset(&a, 0, sizeof(a));
    a.o = o.p;
    a.heads = heads;
    a.head_dim = o.C / heads;
    a.scale = 1.0f / std::sqrt(static_cast<float>(a.head_dim));
    a.kv_batch_div = 1;
    a.b_inner = 1;
    return a;
}

void attn_step(Ctx& c, const AttnParams& a, const char* label) {
    c.b->step([a](cudaStream_t s) { return attention(a, s); }, 1, STEP_ATTN,
              4.0 * a.batch * a.heads * static_cast<double>(a.sq) * a.skv * a.head_dim, label);
}

// the fused q|k|v projection of a self-attention
Tok qkv_proj(Ctx& c, const Tok& x, const std::string& ap, const std::string& lnp) {
    const __half* w = w_cat(c, {ap + ".to_q.weight", ap + ".to_k.weight", ap + ".to_v.weight"});
    return ln_linear(c, x, lnp, ap + ".qkv", w, nullptr, 3 * x.C, nullptr);
}

// after the attention that read `in` and wrote o: x + to_out(o)
Tok attn_out(Ctx& c, const Tok& x, const Tok& o, const Tok& in, const std::string& ap) {
    c.b->free(in);
    Tok y = linear(c, o, prm(c, ap + ".to_out.0.weight"), x.C, prm(c, ap + ".to_out.0.bias"), &x);
    c.b->free(o);
    c.b->free(x);
    return y;
}

// spatial self-attention: every sequence is the P tokens of one frame
Tok attn_spatial(Ctx& c, const Tok& x, const std::string& ap, const std::string& lnp, int heads, long long P, const char* label) {
    const int C = x.C;
    Tok o = c.b->alloc(x.rows, C);
    Tok qkv = qkv_proj(c, x, ap, lnp);
    AttnParams a = attn_params(o, heads);
    a.q = qkv.p;
    a.k = qkv.p + C;
    a.v = qkv.p + 2 * C;
    a.batch = static_cast<int>(x.rows / P);
    a.sq = a.skv = static_cast<int>(P);
    a.q_bs = a.k_bs = a.v_bs = P * qkv.ld;
    a.q_ss = a.k_ss = a.v_ss = qkv.ld;
    a.o_bs = P * o.ld;
    a.o_ss = o.ld;
    attn_step(c, a, label);
    return attn_out(c, x, o, qkv, ap);
}

// cross-attention on the prompt, queries as in attn_spatial.  A prompt's K/V are the same for every frame (the reference
// recomputes them per frame, t2v_model.py:426, :545-546; attention_temporal.py:321-325) and, with a context batch Bc < B,
// for every sample sharing it: only the Bc * L context rows are projected.
Tok attn_cross(Ctx& c, const Tok& x, const std::string& ap, const std::string& lnp, int heads, long long P, const char* label) {
    const int C = x.C;
    Tok o = c.b->alloc(x.rows, C);
    Tok q = ln_linear(c, x, lnp, ap + ".to_q", prm(c, ap + ".to_q.weight"), nullptr, C, nullptr);
    Tok ctx_tok;
    ctx_tok.p = c.ctx;
    ctx_tok.rows = static_cast<long long>(c.Bc) * c.L;
    ctx_tok.C = c.u->cfg.context_dim;
    ctx_tok.ld = ctx_tok.C;
    const __half* wkv = w_cat(c, {ap + ".to_k.weight", ap + ".to_v.weight"});
    Tok kv = linear(c, ctx_tok, wkv, 2 * C, nullptr, nullptr);
    AttnParams a = attn_params(o, heads);
    a.q = q.p;
    a.k = kv.p;
    a.v = kv.p + C;
    a.batch = static_cast<int>(x.rows / P);
    a.sq = static_cast<int>(P);
    a.skv = c.L;
    a.q_bs = P * q.ld;
    a.q_ss = q.ld;
    a.k_bs = a.v_bs = static_cast<long long>(c.L) * kv.ld;
    a.k_ss = a.v_ss = kv.ld;
    // frames per prompt IN THIS MATRIX: frames per sample (frame-sharded clip: this rank's frames) x samples per prompt
    a.kv_batch_div = c.Fl * (c.B / c.Bc);
    a.o_bs = P * o.ld;
    a.o_ss = o.ld;
    attn_step(c, a, label);
    c.b->free(kv);
    return attn_out(c, x, o, q, ap);
}

// ModelScope's temporal self-attention (TemporalTransformer, t2v_model.py:684-685): a sequence runs along the F frames of
// one pixel.  Rows (b, f, pixel) with P pixels per frame: in a sharded clip, this rank's pixels of the pixel-sharded layout.
Tok attn_temporal(Ctx& c, const Tok& x, const std::string& ap, const std::string& lnp, int heads, long long P) {
    const int C = x.C;
    Tok o = c.b->alloc(x.rows, C);
    Tok qkv = qkv_proj(c, x, ap, lnp);
    AttnParams a = attn_params(o, heads);
    a.q = qkv.p;
    a.k = qkv.p + C;
    a.v = qkv.p + 2 * C;
    a.batch = static_cast<int>(c.B * P);
    a.b_inner = static_cast<int>(P);
    a.sq = a.skv = c.F;
    a.q_bs = a.k_bs = a.v_bs = static_cast<long long>(c.F) * P * qkv.ld;
    a.q_bsi = a.k_bsi = a.v_bsi = qkv.ld;
    a.q_ss = a.k_ss = a.v_ss = P * qkv.ld;
    a.o_bs = static_cast<long long>(c.F) * P * o.ld;
    a.o_bsi = o.ld;
    a.o_ss = P * o.ld;
    attn_step(c, a, "attn temporal");
    return attn_out(c, x, o, qkv, ap);
}

// VideoCrafter's temporal self-attention with relative-position K/V tables (TemporalCrossAttention, RelativePosition,
// attention_temporal.py:46-65, :107-144): the sequences of attn_temporal; the FLOP count adds 2 * max_rel + 1 keys for the
// two table products
Tok attn_relpos(Ctx& c, const Tok& x, const std::string& ap, const std::string& lnp, int heads, long long P) {
    const int C = x.C, d = C / heads;
    Tok o = c.b->alloc(x.rows, C);
    Tok qkv = qkv_proj(c, x, ap, lnp);
    RelposParams r;
    memset(&r, 0, sizeof(r));
    r.q = qkv.p;
    r.k = qkv.p + C;
    r.v = qkv.p + 2 * C;
    r.o = o.p;
    r.table_k = prm(c, ap + ".relative_position_k.embeddings_table");
    r.table_v = prm(c, ap + ".relative_position_v.embeddings_table");
    r.n_seq = static_cast<long long>(c.B) * P;
    r.seq_inner = P;
    r.bs_outer = static_cast<long long>(c.F) * P * qkv.ld;
    r.bs_inner = qkv.ld;
    r.ss = P * qkv.ld;
    r.o_bs_outer = static_cast<long long>(c.F) * P * o.ld;
    r.o_bs_inner = o.ld;
    r.o_ss = P * o.ld;
    r.heads = heads;
    r.head_dim = d;
    r.T = c.F;
    r.max_rel = c.u->cfg.temporal_length;
    r.scale = 1.0f / std::sqrt(static_cast<float>(d));
    const int nrel = 2 * r.max_rel + 1;
    c.b->step([r](cudaStream_t s) { return attention_relpos(r, s); }, 1, STEP_ATTN,
              4.0 * r.n_seq * heads * static_cast<double>(c.F) * (c.F + nrel) * d, "attn temporal relpos (vc)");
    return attn_out(c, x, o, qkv, ap);
}

// GEGLU feed-forward (t2v_model.py:813-821, :833-846): x + net.2(GEGLU(net.0.proj(LN x))), the GEGLU fused into the first
// GEMM's epilogue.  Its packed weight interleaves the two halves per tile, so the tile width is fixed here.
Tok feed_forward(Ctx& c, const Tok& x, const std::string& p) {
    const int C = x.C, H = 4 * C;
    const int bn = (2 * H) % 256 == 0 ? 256 : ((2 * H) % 128 == 0 ? 128 : 64);
    Geglu g = w_geglu(c, p + ".ff.net.0.proj", H, C, bn);
    Tok gg = ln_linear(c, x, p + ".norm3", p + ".ff.net.0.proj#geglu" + std::to_string(bn), g.w, g.b, 2 * H, nullptr, GEMM_GEGLU, bn);
    Tok y = linear(c, gg, prm(c, p + ".ff.net.2.weight"), C, prm(c, p + ".ff.net.2.bias"), &x);
    c.b->free(gg);
    c.b->free(x);
    return y;
}

// GroupNorm -> proj_in -> transformer block -> proj_out + x, all on the one token matrix [(b, f, y, x), C] (none of the
// reference's rearranges exist).  The block:
//   ST  SpatialTransformer (t2v_model.py:639-658, use_linear): spatial self -> cross -> FF;
//   TT  TemporalTransformer (:716-767, Conv1d k=1 projections): temporal self twice (only_self_att, :684-685) -> FF;
//   STT VideoCrafter's SpatialTemporalTransformer (attention_temporal.py:386-399): spatial self -> relpos temporal ->
//       cross -> relpos temporal again ("attn2_tmp" with context None) -> FF.
Tok transformer(Ctx& c, const Tok& x, const Blk& blk, int hcur, int wcur) {
    // TT: rows (b, f, own pixels) -- all frames local; the 5-D GroupNorm's statistics span every rank's pixels
    const bool temporal = blk.kind == Blk::TT;
    const long long Pfull = static_cast<long long>(hcur) * wcur;
    const long long P = temporal ? own_pixels(c, hcur, wcur) : Pfull;
    const std::string& p = blk.prefix;
    Tok n = group_norm(c, x, p + ".norm", temporal ? P * c.F : norm_rows(c, P), 1e-6f, false,
                       (temporal && c.nranks > 1) ? Pfull * c.F : 0);
    Tok h = linear(c, n, prm(c, p + ".proj_in.weight"), blk.inner, prm(c, p + ".proj_in.bias"), nullptr);
    c.b->free(n);
    const std::string t = p + ".transformer_blocks.0";
    const int heads = blk.heads;
    switch (blk.kind) {
        case Blk::ST:
            h = attn_spatial(c, h, t + ".attn1", t + ".norm1", heads, P, "attn spatial");
            h = attn_cross(c, h, t + ".attn2", t + ".norm2", heads, P, "attn cross");
            break;
        case Blk::TT:
            h = attn_temporal(c, h, t + ".attn1", t + ".norm1", heads, P);
            h = attn_temporal(c, h, t + ".attn2", t + ".norm2", heads, P);
            break;
        default:        // Blk::STT
            h = attn_spatial(c, h, t + ".attn1", t + ".norm1", heads, P, "attn spatial (vc)");
            h = attn_relpos(c, h, t + ".attn1_tmp", t + ".norm4", heads, P);
            h = attn_cross(c, h, t + ".attn2", t + ".norm2", heads, P, "attn cross (vc)");
            h = attn_relpos(c, h, t + ".attn2_tmp", t + ".norm5", heads, P);
            break;
    }
    h = feed_forward(c, h, t);
    Tok y = linear(c, h, prm(c, p + ".proj_out.weight"), blk.cin, prm(c, p + ".proj_out.bias"), &x);
    c.b->free(h);
    return y;
}

// ResBlock._forward (t2v_model.py:983-1009; VideoCrafter openaimodel3d.py:244-271, whose Conv3d (1,3,3) are the same
// per-frame 3x3 convs), then ModelScope's TemporalConvBlock_v2.forward (:1218-1229)
Tok res_block(Ctx& c, const Tok& x, const Blk& blk, int hcur, int wcur) {
    const std::string& p = blk.prefix;
    const long long P = static_cast<long long>(hcur) * wcur;
    const int Co = blk.cout;
    const int E = c.u->cfg.dim * 4;
    // emb_layers(SiLU -> Linear) per sample, folded with conv1's bias into a per-sample bias row
    __half* bias1 = reinterpret_cast<__half*>(c.b->alloc_bytes(static_cast<size_t>(c.B) * Co * sizeof(__half)));
    {
        const __half* we = prm(c, p + ".emb_layers.1.weight");
        const __half* be = prm(c, p + ".emb_layers.1.bias");
        const __half* bc = prm(c, p + ".in_layers.2.bias");
        const __half* emb = c.emb;
        const int B = c.B;
        c.b->step([=](cudaStream_t s) { return small_linear(emb, E, we, be, bc, bias1, Co, B, Co, E, 1, s); });
    }
    Tok a = group_norm(c, x, p + ".in_layers.0", norm_rows(c, P), 1e-5f, true);
    Tok h = conv3x3(c, a, p + ".in_layers.2.weight", bias1, static_cast<int>(c.Fl * P), Co, Co, hcur, wcur, nullptr);
    c.b->free(a);
    Tok bn_ = group_norm(c, h, p + ".out_layers.0", norm_rows(c, P), 1e-5f, true);
    c.b->free(h);
    Tok skip = x;
    bool own_skip = false;
    if (blk.cin != blk.cout) {
        skip = linear(c, x, prm(c, p + ".skip_connection.weight"), Co, prm(c, p + ".skip_connection.bias"), nullptr);
        own_skip = true;
    }
    Tok h2 = conv3x3(c, bn_, p + ".out_layers.3.weight", prm(c, p + ".out_layers.3.bias"), 0, 0, Co, hcur, wcur, &skip);
    c.b->free(bn_);
    if (own_skip) c.b->free(skip);
    c.b->free_bytes(bias1);
    if (c.u->cfg.arch == 1) return h2;
    // temporal conv block: 4 x [GN(5-D: statistics over all frames of a sample) -> SiLU -> Conv3d (3,1,1)] + identity.
    // Sharded clip: transpose to the pixel-sharded layout first -- all F frames of this rank's pixels are then local, the
    // 3-tap conv and its zero padding at f = 0, F-1 need no halo; only the GroupNorm sums cross ranks.
    const long long Pt = own_pixels(c, hcur, wcur);
    if (c.nranks > 1) {
        Tok hp = exchange(c, h2, true, hcur, wcur);
        c.b->free(h2);
        h2 = hp;
    }
    const long long Rt = h2.rows;
    const char* names[4] = {"conv1", "conv2", "conv3", "conv4"};
    const int idx[4] = {2, 3, 3, 3};
    Tok y = h2;
    for (int i = 0; i < 4; ++i) {
        const std::string tp = p + ".temopral_conv." + names[i];
        Tok g = group_norm(c, y, tp + ".0", Pt * c.F, 1e-5f, true, c.nranks > 1 ? P * c.F : 0);
        const std::string wn = tp + "." + std::to_string(idx[i]);
        const __half* w = w_conv(c, wn + ".weight", 3);
        Tok y2 = c.b->alloc(Rt, Co);
        GemmProblem pr = base_problem(g, Co, w, Co, Co, y2);
        pr.nd = 3;
        pr.dim[0] = static_cast<int>(Pt);
        pr.dim[1] = c.F;
        pr.dim[2] = c.B;
        taps_temporal(pr);
        pr.bias = prm(c, wn + ".bias");
        if (i == 3) {
            pr.residual = h2.p;
            pr.ldr = h2.ld;
        }
        c.b->gemm(pr);
        c.b->free(g);
        if (i > 0) c.b->free(y);
        y = y2;
    }
    c.b->free(h2);
    return y;
}

Tok downsample(Ctx& c, const Tok& x, const Blk& blk, int hcur, int wcur) {
    const int frames = static_cast<int>(x.rows / (static_cast<long long>(hcur) * wcur));
    const int ho = (hcur + 1) / 2, wo = (wcur + 1) / 2;
    Tok col = c.b->alloc(static_cast<long long>(frames) * ho * wo, 9 * x.C);
    const Tok xx = x;
    c.b->step([=](cudaStream_t s) { return im2col_s2(xx.p, col.p, frames, hcur, wcur, xx.C, s); });
    const __half* w = w_conv_kmajor(c, blk.prefix + ".op.weight");
    Tok y = linear(c, col, w, blk.cout, prm(c, blk.prefix + ".op.bias"), nullptr);
    c.b->free(col);
    return y;
}

Tok upsample(Ctx& c, const Tok& x, const Blk& blk, int hcur, int wcur) {
    const int frames = static_cast<int>(x.rows / (static_cast<long long>(hcur) * wcur));
    Tok u = c.b->alloc(x.rows * 4, x.C);
    const Tok xx = x;
    c.b->step([=](cudaStream_t s) { return upsample2x(xx.p, u.p, frames, hcur, wcur, xx.C, s); });
    Tok y = conv3x3(c, u, blk.prefix + ".conv.weight", prm(c, blk.prefix + ".conv.bias"), 0, 0, blk.cout, 2 * hcur,
                    2 * wcur, nullptr);
    c.b->free(u);
    return y;
}

// input blocks after which VideoCrafter's UNetModel adds an adapter feature (openaimodel3d.py:658): (id + 1) % 3 == 0
bool feature_block(int id) { return (id + 1) % 3 == 0; }
int n_feature_blocks(const t2v_unet* u) {
    int n = 0;
    for (size_t id = 0; id < u->ins.size(); ++id) n += feature_block(static_cast<int>(id)) ? 1 : 0;
    return n;
}

// feats_B > 0: the plan variant with adapter features (VideoCrafter only), staged for feats_B samples.
// Bc: context batch (B % Bc == 0), the prompts staged and projected for the cross-attentions.
int build(t2v_unet* u, Plan* plan, Arena* arena, bool dry, cudaStream_t stream, int B, int Bc, int F, int h, int w, int L,
          IO* io, int feats_B = 0) {
    Builder bld(plan, arena, dry, num_sms());
    Ctx c;
    c.params = &u->params;
    c.b = &bld;
    c.stream = stream;
    c.gn_ws = u->gn_ws.ptr;
    c.u = u;
    c.B = B; c.Bc = Bc; c.F = F; c.h = h; c.w = w; c.L = L;
    c.emb = nullptr; c.ctx = nullptr; c.plan = plan;
    c.Fl = F; c.rank = 0; c.nranks = 1; c.slab = plan->slab;
    const bool sharded = u->shard_on && plan->shard != nullptr;
    if (sharded) {                       // this rank's frames of the clip; temporal modules see all F of its pixel range
        c.rank = u->peers.rank;
        c.nranks = u->peers.nranks;
        c.Fl = plan->shard->fb[c.rank + 1] - plan->shard->fb[c.rank];
        c.shard_peers = &u->peers;
        c.plan_shard = plan->shard.get();
        plan->shard->n_xchg = 0;
        plan->shard->n_gn = 0;
        if (!dry) {
            ShardComm* comm = u->comm;
            bld.step([comm](cudaStream_t s) { return shard_bump_epoch(comm, s); }, 1, STEP_OTHER, 0.0, "epoch");
        }
    }
    const t2v_unet_config& cfg = u->cfg;
    const int E = cfg.dim * 4;
    const long long R0 = static_cast<long long>(B) * c.Fl * h * w;
    const int cin_pad = round_up(cfg.in_dim, 8);

    // fixed I/O staging at the head of the slab (graph-replay friendly)
    Tok x0 = bld.alloc(R0, cin_pad);
    io->x_tok = x0.p;
    io->t = reinterpret_cast<float*>(bld.alloc_bytes(static_cast<size_t>(B) * sizeof(float)));
    Tok ctx_tok = bld.alloc(static_cast<long long>(Bc) * L, cfg.context_dim);
    c.ctx = ctx_tok.p;
    io->ctx = ctx_tok.p;
    io->n_feat = 0;
    if (feats_B > 0) {                   // feature staging, filled per forward like ctx; level sizes follow the input blocks
        int hf = h, wf = w;
        for (size_t id = 0; id < u->ins.size(); ++id) {
            const Blk& b0 = u->ins[id][0];
            if (b0.kind == Blk::DOWN) {
                hf = (hf + 1) / 2;
                wf = (wf + 1) / 2;
            }
            if (!feature_block(static_cast<int>(id))) continue;
            if (io->n_feat >= kMaxFeat) {
                set_error("more than %d adapter injection points", kMaxFeat);
                return -7;
            }
            const int Cf = u->ins[id].back().cout;
            Tok f = bld.alloc(static_cast<long long>(feats_B) * F * hf * wf, Cf);
            io->feat[io->n_feat] = f.p;
            io->feat_elems[io->n_feat] = f.rows * f.C;
            io->n_feat += 1;
        }
    }
    // time embedding: sinusoid -> Linear -> SiLU -> Linear (t2v_model.py:154-156, :420)
    __half* sinus = reinterpret_cast<__half*>(bld.alloc_bytes(static_cast<size_t>(B) * cfg.dim * sizeof(__half)));
    __half* e1 = reinterpret_cast<__half*>(bld.alloc_bytes(static_cast<size_t>(B) * E * sizeof(__half)));
    __half* e2 = reinterpret_cast<__half*>(bld.alloc_bytes(static_cast<size_t>(B) * E * sizeof(__half)));
    c.emb = e2;
    {
        const float* tp = io->t;
        const int dim = cfg.dim;
        const __half* w0 = prm(c, "time_embed.0.weight");
        const __half* b0 = prm(c, "time_embed.0.bias");
        const __half* w2 = prm(c, "time_embed.2.weight");
        const __half* b2 = prm(c, "time_embed.2.bias");
        bld.step([=](cudaStream_t s) { return time_sinusoid(tp, sinus, B, dim, s); });
        bld.step([=](cudaStream_t s) { return small_linear(sinus, dim, w0, b0, nullptr, e1, E, B, E, dim, 0, s); });
        bld.step([=](cudaStream_t s) { return small_linear(e1, E, w2, b2, nullptr, e2, E, B, E, E, 1, s); });
    }

    int hc = h, wc = w;
    std::vector<Tok> xs;
    std::vector<std::pair<int, int>> xs_hw;
    Tok x = x0;
    bool x_is_io = true;
    bool x_ps = false;                   // sharded clip: x is in the pixel-sharded layout (after a temporal module)
    // x is released unless it is a pending skip connection or the I/O staging buffer
    auto release = [&](const Tok& t) {
        for (const Tok& s : xs)
            if (s.p == t.p) return;
        if (t.p == x0.p && x_is_io) return;
        bld.free(t);
    };
    // sharded clip: bring x into the layout the next module works in (spatial modules: frame-sharded, temporal: pixel-sharded)
    auto to_layout = [&](bool want_ps) {
        if (!sharded || x_ps == want_ps) return;
        Tok y = exchange(c, x, want_ps, hc, wc);
        release(x);
        x_is_io = false;
        x = y;
        x_ps = want_ps;
    };
    auto run_block = [&](const std::vector<Blk>& blk) {
        for (const Blk& b : blk) {
            Tok y;
            to_layout(b.kind == Blk::TT);
            switch (b.kind) {
                case Blk::STEM:
                    y = conv3x3(c, x, b.prefix + ".weight", prm(c, b.prefix + ".bias"), 0, 0, b.cout, hc, wc, nullptr);
                    break;
                case Blk::RES: y = res_block(c, x, b, hc, wc); break;
                case Blk::ST:
                case Blk::TT:
                case Blk::STT: y = transformer(c, x, b, hc, wc); break;
                case Blk::DOWN:
                    y = downsample(c, x, b, hc, wc);
                    hc = (hc + 1) / 2;
                    wc = (wc + 1) / 2;
                    break;
                case Blk::UP:
                    y = upsample(c, x, b, hc, wc);
                    hc *= 2;
                    wc *= 2;
                    break;
            }
            if (sharded && b.kind == Blk::RES) x_ps = true;     // res_block ends in the temporal conv block (pixel-sharded)
            if (sharded && x_ps) tap(c, b.prefix, y, 1, own_pixels(c, hc, wc));      // pixel-sharded: rows (b, f, own pixel)
            else tap(c, b.prefix, y, hc, wc);
            release(x);
            x_is_io = false;
            x = y;
        }
    };
    int feat_i = 0;
    for (size_t id = 0; id < u->ins.size(); ++id) {
        run_block(u->ins[id]);
        to_layout(false);                // skip connections (and the next block's ResBlock) are frame-sharded
        if (feats_B > 0 && feature_block(static_cast<int>(id))) {       // h = h + features_adapter[i], before the push
            const Tok xx = x;
            if (u->taps_enabled) {       // the add is in place: the block's tap keeps a copy of its output from before it
                const Tok snap = bld.alloc(xx.rows, xx.C);
                bld.step([=](cudaStream_t s) {
                    if (cudaMemcpy2DAsync(snap.p, snap.ld * sizeof(__half), xx.p, xx.ld * sizeof(__half), xx.C * sizeof(__half),
                                          xx.rows, cudaMemcpyDeviceToDevice, s) != cudaSuccess)
                        return launch_status("feature tap copy");
                    return 0;
                });
                tap(c, u->ins[id].back().prefix, snap, hc, wc);
            }
            const __half* f = io->feat[feat_i++];
            const long long per_sample = static_cast<long long>(F) * hc * wc;
            const int fb = feats_B;
            bld.step([=](cudaStream_t s) { return feature_add(xx.p, xx.ld, f, xx.C, xx.rows, per_sample, fb, s); }, 1, STEP_OTHER,
                     0.0, "adapter feature add");
        }
        xs.push_back(x);
        xs_hw.push_back({hc, wc});
    }
    run_block(u->mid);
    for (auto& blk : u->outs) {
        to_layout(false);
        Tok skip = xs.back();
        xs.pop_back();
        xs_hw.pop_back();
        Tok cat = bld.alloc(x.rows, x.C + skip.C);
        {
            const Tok xa = x, sb = skip;
            bld.step([=](cudaStream_t s) {
                return concat_cols(xa.p, xa.ld, xa.C, sb.p, sb.ld, sb.C, cat.p, cat.ld, xa.rows, s);
            });
        }
        // x (output of the previous block) may itself still be on the skip stack only in the encoder; here it is free
        bool x_on_stack = false;
        for (const Tok& s : xs)
            if (s.p == x.p) x_on_stack = true;
        if (!x_on_stack && x.p != skip.p) bld.free(x);
        bld.free(skip);
        x = cat;
        run_block(blk);
    }
    to_layout(false);
    // head: GN -> SiLU -> Conv3x3 dim -> out_dim (t2v_model.py:321-323)
    Tok g = group_norm(c, x, "out.0", norm_rows(c, static_cast<long long>(hc) * wc), 1e-5f, true);
    bld.free(x);
    Tok o = conv3x3(c, g, "out.2.weight", prm(c, "out.2.bias"), 0, 0, cfg.out_dim, hc, wc, nullptr, 16);
    bld.free(g);
    io->out_tok = o.p;
    tap(c, "out", o, hc, wc);
    return bld.error;
}

// The plan-cache key of a forward shape.  The adapter-feature variant adds its feature batch and a shared context its
// context batch Bc < B (a forward without features, one prompt per sample, keeps its plan and key).
std::string plan_key(const t2v_unet* u, int B, int Bc, int F, int h, int w, int L, int feats_B) {
    char key[128];
    snprintf(key, sizeof(key), "%d,%d,%d,%d,%d,%d,%d/%d", B, F, h, w, L, u->taps_enabled ? 1 : 0, u->shard_on ? u->peers.rank : 0,
             u->shard_on ? u->peers.nranks : 1);
    if (feats_B > 0) {
        const size_t n = strlen(key);
        snprintf(key + n, sizeof(key) - n, ",a%d", feats_B);
    }
    if (Bc != B) {
        const size_t n = strlen(key);
        snprintf(key + n, sizeof(key) - n, ",c%d", Bc);
    }
    return key;
}

// The frame partition of a sharded clip of F frames (null when the denoiser is not sharded).
std::shared_ptr<PlanShard> new_plan_shard(const t2v_unet* u, int F) {
    if (!u->shard_on) return nullptr;
    std::shared_ptr<PlanShard> s(new PlanShard());
    s->own_rank = u->peers.rank;
    shard_partition(F, u->peers.nranks, s->fb);
    return s;
}

PlanCache<IO>::Entry* get_plan(t2v_unet* u, int B, int Bc, int F, int h, int w, int L, cudaStream_t stream, int feats_B = 0) {
    const std::string key = plan_key(u, B, Bc, F, h, w, L, feats_B);
    if (auto* e = u->plans.find(key, u->params.version())) return e;
    if (!u->params.complete("UNet")) return nullptr;
    // groupnorm workspace: the largest (rows_per_inst, n_inst) pair is the per-sample 5-D norm at level 0
    size_t need = std::max(gn_workspace_bytes(F * h * w, B, num_sms()), gn_workspace_bytes(h * w, B * F, num_sms()));
    need = std::max(need, gn_workspace_bytes(1, B * F, num_sms()));
    if (u->gn_ws.ensure(need + (1 << 20), stream)) u->plans.clear(stream);
    if (!u->gn_ws.ptr) return nullptr;
    if (u->shard_on) {
        if (u->cfg.arch != 0) {
            set_error("frame sharding is built for the ModelScope UNetSD (arch 0)");
            return nullptr;
        }
        int deepest = h * w;
        for (int i = 1; i < u->cfg.n_mult; ++i) deepest = ((h + (1 << i) - 1) >> i) * ((w + (1 << i) - 1) >> i);
        if (F < u->peers.nranks || deepest < u->peers.nranks || B > SHARD_MAX_INST) {
            set_error("frame sharding over %d ranks needs >= %d frames, >= %d pixels at the deepest level (got %d) and B <= %d",
                      u->peers.nranks, u->peers.nranks, u->peers.nranks, deepest, SHARD_MAX_INST);
            return nullptr;
        }
    }
    std::unique_ptr<Plan> shell(new Plan());
    shell->shard = new_plan_shard(u, F);
    return u->plans.build(key, u->params.version(), stream, std::move(shell),
                          u->taps_enabled || getenv("T2V_ARENA_NO_REUSE") != nullptr, "UNet",
                          [&](Plan* p, Arena* a, bool dry, IO* io) { return build(u, p, a, dry, stream, B, Bc, F, h, w, L, io, feats_B); });
}

// A tap of the most recently used plan: (tokens, (h, w)); null, with the error set, if that plan has no such tap.
const std::pair<Tok, std::pair<int, int>>* find_tap(t2v_unet* u, const char* name) {
    auto* entry = u->plans.latest();
    if (entry) {
        auto it = entry->plan->taps.find(name);
        if (it != entry->plan->taps.end()) return &it->second;
    }
    set_error("tap '%s' not found (enable taps before the forward)", name);
    return nullptr;
}

}  // namespace
}  // namespace t2v

extern "C" {

int t2v_unet_create(const t2v_unet_config* cfg, t2v_unet** out) {
    if (!cfg || !out) return -1;
    if (cfg->arch == 0 && cfg->head_dim != 64) {
        set_error("head_dim must be 64 (got %d)", cfg->head_dim);
        return -2;
    }
    if (cfg->dim % 64 != 0 || cfg->context_dim % 8 != 0) {
        set_error("dim must be a multiple of 64 and context_dim of 8");
        return -2;
    }
    if (cfg->arch == 1 && (cfg->num_heads < 1 || (cfg->dim / cfg->num_heads) % 8 != 0 || cfg->temporal_length < 1 ||
                           2 * cfg->temporal_length + 1 > 48)) {
        set_error("VideoCrafter UNetModel: head width dim/num_heads must be a multiple of 8 and temporal_length <= 23");
        return -2;
    }
    if (cfg->arch != 0 && cfg->arch != 1) {
        set_error("unknown arch %d", cfg->arch);
        return -2;
    }
    t2v_unet* u = new t2v_unet();
    u->cfg = *cfg;
    if (cfg->arch == 1) {
        enumerate_vc(u);
        expect_params_vc(u);
    } else {
        enumerate(u);
        expect_params(u);
    }
    *out = u;
    return 0;
}

void t2v_unet_destroy(t2v_unet* u) { delete u; }

int t2v_unet_set_param(t2v_unet* u, const char* name, const void* data, int dtype, int ndim, const int64_t* shape,
                       void* stream) {
    return u->params.set(name, data, dtype, ndim, shape, reinterpret_cast<cudaStream_t>(stream));
}

int t2v_unet_missing_params(t2v_unet* u, char* name_out, size_t name_cap) { return missing_params_out(u->params, name_out, name_cap); }

int t2v_unet_param_info(t2v_unet* u, int index, char* name_out, size_t name_cap, int64_t* shape_out, int* ndim_out) {
    return param_info_out(u->params, index, name_out, name_cap, shape_out, ndim_out);
}

}  // extern "C"

namespace t2v {
namespace {

int check_ctx_batch(const t2v_unet* u, int B, int ctx_B) {
    if (ctx_B < 1 || B < 1 || B % ctx_B != 0) {
        set_error("context batch %d does not divide the forward batch %d", ctx_B, B);
        return -2;
    }
    if (u->shard_on && ctx_B != B) {
        set_error("a shared context batch (%d prompts for %d samples) is not built for the frame-sharded denoiser", ctx_B, B);
        return -2;
    }
    return 0;
}

int unet_forward(t2v_unet* u, const void* x, int x_is_f32, const float* t, const void* ctx, int ctx_B, const void* const* feats,
                 int feats_B, void* out, int out_is_f32, int B, int F, int h, int w, int L, cudaStream_t stream) {
    if (u->cfg.arch == 1 && F > 32) {
        set_error("VideoCrafter temporal attention kernel: at most 32 frames per clip (got %d)", F);
        return -4;
    }
    auto* entry = get_plan(u, B, ctx_B, F, h, w, L, stream, feats_B);
    if (!entry) return -1;
    Plan* plan = entry->plan.get();
    const IO& io = entry->io;
    const t2v_unet_config& cfg = u->cfg;
    const int cin_pad = (cfg.in_dim + 7) / 8 * 8;
    if (u->shard_on) {                   // x / out hold this rank's frames only: [B, C, F_local, h, w]
        if (!plan->shard->connected) {
            set_error("frame-sharded forward before t2v_unet_shard_connect for this shape");
            return -5;
        }
        F = plan->shard->fb[u->peers.rank + 1] - plan->shard->fb[u->peers.rank];
    }
    int rc = ingest_latent(x, x_is_f32, io.x_tok, cin_pad, cin_pad, B, cfg.in_dim, F, h, w, 1.0f, stream);
    if (rc != 0) return rc;
    cudaMemcpyAsync(io.t, t, sizeof(float) * B, cudaMemcpyDeviceToDevice, stream);
    cudaMemcpyAsync(io.ctx, ctx, static_cast<size_t>(ctx_B) * L * cfg.context_dim * sizeof(__half), cudaMemcpyDeviceToDevice,
                    stream);
    for (int i = 0; i < io.n_feat; ++i)
        cudaMemcpyAsync(io.feat[i], feats[i], static_cast<size_t>(io.feat_elems[i]) * sizeof(__half), cudaMemcpyDeviceToDevice, stream);
    rc = run_plan(plan, stream, !u->taps_enabled);
    if (rc != 0) {
        set_error("UNet launch failed (%d): %s", rc, cudaGetErrorString(cudaGetLastError()));
        return rc;
    }
    u->last_launches = plan->launches + 2;
    u->last_exchanges = plan->shard ? plan->shard->n_xchg : 0;
    const int out_ld = (cfg.out_dim % 8 == 0) ? cfg.out_dim : (cfg.out_dim + 7) / 8 * 8;
    return egress_latent(io.out_tok, out_ld, out, out_is_f32, B, cfg.out_dim, F, h, w, stream);
}

}  // namespace
}  // namespace t2v

extern "C" {

int t2v_unet_forward(t2v_unet* u, const void* x, int x_is_f32, const float* t, const void* ctx, void* out,
                     int out_is_f32, int B, int F, int h, int w, int L, void* stream_) {
    clear_pending_error("t2v_unet_forward");
    return unet_forward(u, x, x_is_f32, t, ctx, B, nullptr, 0, out, out_is_f32, B, F, h, w, L, reinterpret_cast<cudaStream_t>(stream_));
}

int t2v_unet_forward_ctx(t2v_unet* u, const void* x, int x_is_f32, const float* t, const void* ctx, int ctx_B, void* out,
                         int out_is_f32, int B, int F, int h, int w, int L, void* stream_) {
    clear_pending_error("t2v_unet_forward_ctx");
    if (const int rc = check_ctx_batch(u, B, ctx_B)) return rc;
    return unet_forward(u, x, x_is_f32, t, ctx, ctx_B, nullptr, 0, out, out_is_f32, B, F, h, w, L,
                        reinterpret_cast<cudaStream_t>(stream_));
}

int t2v_unet_forward_adapter(t2v_unet* u, const void* x, int x_is_f32, const float* t, const void* ctx,
                             const void* const* feats, int n_feats, int feats_B, void* out, int out_is_f32, int B, int F, int h,
                             int w, int L, void* stream_) {
    clear_pending_error("t2v_unet_forward_adapter");
    if (u->cfg.arch != 1) {
        set_error("adapter features are a VideoCrafter UNetModel input (arch 1); this denoiser is arch %d", u->cfg.arch);
        return -2;
    }
    const int want = n_feature_blocks(u);
    if (n_feats != want) {
        set_error("adapter features: got %d feature maps, the UNet adds one after each of its %d input blocks with (id + 1) %% 3 == 0",
                  n_feats, want);
        return -2;
    }
    if (feats_B < 1 || B % feats_B != 0) {
        set_error("adapter features: feature batch %d does not divide the forward batch %d", feats_B, B);
        return -2;
    }
    if (feats == nullptr) {
        set_error("adapter features: null feature list");
        return -2;
    }
    for (int i = 0; i < n_feats; ++i)
        if (feats[i] == nullptr) {
            set_error("adapter features: feature %d is a null pointer", i);
            return -2;
        }
    return unet_forward(u, x, x_is_f32, t, ctx, B, feats, feats_B, out, out_is_f32, B, F, h, w, L, reinterpret_cast<cudaStream_t>(stream_));
}

double t2v_unet_flops(t2v_unet* u, int B, int F, int h, int w, int L) {
    IO io;
    double flops = 0.0;
    // a sharded denoiser counts this rank's share of the clip's work
    if (dry_build(new_plan_shard(u, F), false, [&](Plan* p, Arena* a, bool dry) { return build(u, p, a, dry, nullptr, B, B, F, h, w, L, &io); },
                  &flops) < 0)
        return -1.0;
    return flops;
}

int t2v_unet_plan_bytes(t2v_unet* u, int B, int F, int h, int w, int L, size_t* arena) {
    return t2v_unet_plan_info(u, B, B, F, h, w, L, arena, nullptr, nullptr);
}

int t2v_unet_plan_info(t2v_unet* u, int B, int ctx_B, int F, int h, int w, int L, size_t* arena, double* flops, int* cached) {
    if (!u || !arena) return -1;
    if (const int rc = check_ctx_batch(u, B, ctx_B)) return rc;
    if (cached) *cached = u->plans.holds(plan_key(u, B, ctx_B, F, h, w, L, 0), u->params.version()) ? 1 : 0;
    IO io;
    const long long peak = dry_build(
        new_plan_shard(u, F), false, [&](Plan* p, Arena* a, bool dry) { return build(u, p, a, dry, nullptr, B, ctx_B, F, h, w, L, &io); },
        flops);
    if (peak < 0) return -1;
    *arena = plan_slab_bytes(peak);
    return 0;
}

int t2v_unet_num_launches(t2v_unet* u) { return u->last_launches; }

int t2v_unet_profile(t2v_unet* u, int B, int F, int h, int w, int L, void* stream_, double* out13) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    auto* entry = get_plan(u, B, B, F, h, w, L, stream);
    if (!entry) return -1;
    return profile_plan(entry->plan.get(), stream, out13);
}

// ------------------------------------------------------------------------------------------ frame sharding (shard.cuh)
int t2v_unet_shard_setup(t2v_unet* u, int rank, int nranks) {
    if (nranks < 2 || nranks > SHARD_MAX_RANKS || rank < 0 || rank >= nranks) {
        set_error("shard_setup: need 2 <= nranks <= %d and 0 <= rank < nranks (got %d / %d)", SHARD_MAX_RANKS, rank, nranks);
        return -1;
    }
    if (u->cfg.arch != 0) {
        set_error("frame sharding is built for the ModelScope UNetSD (arch 0)");
        return -1;
    }
    if (u->comm == nullptr) {
        if (cudaMalloc(&u->comm, sizeof(ShardComm)) != cudaSuccess || cudaMemset(u->comm, 0, sizeof(ShardComm)) != cudaSuccess) {
            set_error("shard_setup: cudaMalloc of the communication region failed");
            return -2;
        }
    }
    u->plans.clear(nullptr);
    u->peers.rank = rank;
    u->peers.nranks = nranks;
    u->peers.comm[rank] = u->comm;
    u->shard_on = true;
    return 0;
}

int t2v_unet_shard_prepare(t2v_unet* u, int B, int F, int h, int w, int L, void* stream_, t2v_shard_export* out) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!u->shard_on || out == nullptr) {
        set_error("shard_prepare: call t2v_unet_shard_setup first");
        return -1;
    }
    auto* entry = get_plan(u, B, B, F, h, w, L, stream);
    if (!entry) return -1;
    Plan* plan = entry->plan.get();
    memset(out, 0, sizeof(*out));
    static_assert(sizeof(cudaIpcMemHandle_t) <= sizeof(out->comm_handle), "IPC handle size");
    cudaIpcMemHandle_t hc, hs;
    if (cudaIpcGetMemHandle(&hc, u->comm) != cudaSuccess || cudaIpcGetMemHandle(&hs, plan->slab) != cudaSuccess) {
        set_error("shard_prepare: cudaIpcGetMemHandle failed: %s", cudaGetErrorString(cudaGetLastError()));
        return -2;
    }
    memcpy(out->comm_handle, &hc, sizeof(hc));
    memcpy(out->slab_handle, &hs, sizeof(hs));
    out->rank = u->peers.rank;
    out->nranks = u->peers.nranks;
    out->n_exchanges = plan->shard->n_xchg;
    out->n_groupnorms = plan->shard->n_gn;
    for (int k = 0; k < plan->shard->n_xchg; ++k) out->dst_offset[k] = plan->shard->dst_off[k];
    return 0;
}

int t2v_unet_shard_connect(t2v_unet* u, int B, int F, int h, int w, int L, const t2v_shard_export* all, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!u->shard_on || all == nullptr) {
        set_error("shard_connect: call t2v_unet_shard_setup / t2v_unet_shard_prepare first");
        return -1;
    }
    auto* entry = get_plan(u, B, B, F, h, w, L, stream);
    if (!entry) return -1;
    Plan* plan = entry->plan.get();
    PlanShard* ps = plan->shard.get();
    const int me = u->peers.rank, nr = u->peers.nranks;
    for (int r = 0; r < nr; ++r) {
        const t2v_shard_export& e = all[r];
        if (e.rank != r || e.nranks != nr || e.n_exchanges != ps->n_xchg || e.n_groupnorms != ps->n_gn) {
            set_error("shard_connect: export of rank %d does not match this plan (rank %d/%d, %d exchanges, %d norms; here %d, %d)", r,
                      e.rank, e.nranks, e.n_exchanges, e.n_groupnorms, ps->n_xchg, ps->n_gn);
            return -2;
        }
        for (int k = 0; k < ps->n_xchg; ++k) ps->peer_dst_off[r][k] = e.dst_offset[k];
        if (r == me) {
            ps->peer_slab[r] = plan->slab;
            continue;
        }
        if (u->peers.comm[r] == nullptr) {
            cudaIpcMemHandle_t hc;
            memcpy(&hc, e.comm_handle, sizeof(hc));
            void* p = nullptr;
            if (cudaIpcOpenMemHandle(&p, hc, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
                set_error("shard_connect: cudaIpcOpenMemHandle(comm of rank %d) failed: %s", r, cudaGetErrorString(cudaGetLastError()));
                return -3;
            }
            u->peers.comm[r] = reinterpret_cast<ShardComm*>(p);
        }
        if (ps->peer_slab[r] == nullptr) {
            cudaIpcMemHandle_t hs;
            memcpy(&hs, e.slab_handle, sizeof(hs));
            void* p = nullptr;
            if (cudaIpcOpenMemHandle(&p, hs, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) {
                set_error("shard_connect: cudaIpcOpenMemHandle(slab of rank %d) failed: %s", r, cudaGetErrorString(cudaGetLastError()));
                return -3;
            }
            ps->peer_slab[r] = reinterpret_cast<char*>(p);
        }
    }
    ps->connected = true;
    return 0;
}

int t2v_unet_shard_connected(t2v_unet* u, int B, int F, int h, int w, int L) {
    if (!u->shard_on) return 0;
    auto* entry = u->plans.find(plan_key(u, B, B, F, h, w, L, 0), u->params.version());
    return (entry && entry->plan->shard && entry->plan->shard->connected) ? 1 : 0;
}

int t2v_unet_shard_barrier(t2v_unet* u, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    if (!u->shard_on) return -1;
    for (int r = 0; r < u->peers.nranks; ++r)
        if (u->peers.comm[r] == nullptr) {
            set_error("shard_barrier: rank %d is not connected", r);
            return -2;
        }
    int rc = shard_bump_epoch(u->comm, stream);
    if (rc != 0) return rc;
    return shard_barrier(u->peers, SHARD_MAX_XCHG - 1, stream);
}

int t2v_unet_shard_info(t2v_unet* u, int F, int* frame_begin, int* frame_end, int* n_exchanges) {
    if (!u->shard_on) return -1;
    int fb[SHARD_MAX_RANKS + 1];
    shard_partition(F, u->peers.nranks, fb);
    if (frame_begin) *frame_begin = fb[u->peers.rank];
    if (frame_end) *frame_end = fb[u->peers.rank + 1];
    if (n_exchanges) *n_exchanges = u->last_exchanges;
    return 0;
}

// ------------------------------------------------------------------------------------------ LoRA hot-merge
int t2v_unet_lora_merge(t2v_unet* u, const char* weight_name, const void* lora_A, const void* lora_B, int rank, float alpha,
                        int temporal_mean, void* stream) {
    clear_pending_error("t2v_unet_lora_merge");
    return u->params.lora_merge(weight_name, reinterpret_cast<const __half*>(lora_A), reinterpret_cast<const __half*>(lora_B), rank,
                                alpha, temporal_mean, reinterpret_cast<cudaStream_t>(stream));
}

int t2v_unet_lora_apply(t2v_unet* u, const char* weight_name, const void* up, const void* down, int dtype, int rank, float alpha,
                        void* stream) {
    clear_pending_error("t2v_unet_lora_apply");
    return u->params.lora_apply(weight_name, up, down, dtype, rank, alpha, reinterpret_cast<cudaStream_t>(stream));
}

int t2v_unet_lora_restore(t2v_unet* u, const char* weight_name, void* stream) {
    clear_pending_error("t2v_unet_lora_restore");
    return u->params.lora_restore(weight_name, reinterpret_cast<cudaStream_t>(stream));
}

int t2v_unet_lora_clear(t2v_unet* u, void* stream) { return u->params.lora_clear(reinterpret_cast<cudaStream_t>(stream)); }

int t2v_unet_lora_merged(t2v_unet* u) { return u->params.merged_count(); }

int t2v_unet_enable_taps(t2v_unet* u, int on) {
    u->taps_enabled = on != 0;
    return 0;
}

int t2v_unet_tap_info(t2v_unet* u, const char* name, long long* rows, int* C, int* h, int* w) {
    const auto* tap = find_tap(u, name);
    if (!tap) return -1;
    if (rows) *rows = tap->first.rows;
    if (C) *C = tap->first.C;
    if (h) *h = tap->second.first;
    if (w) *w = tap->second.second;
    return 0;
}

long long t2v_unet_read_tap(t2v_unet* u, const char* name, void* dst, long long cap_elems, void* stream_) {
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const auto* tap = find_tap(u, name);
    if (!tap) return -1;
    const Tok& t = tap->first;
    const int h = tap->second.first, w = tap->second.second;
    const long long frames = t.rows / (static_cast<long long>(h) * w);
    const long long n = t.rows * t.C;
    if (n > cap_elems) {
        set_error("tap '%s' needs %lld elements", name, n);
        return -2;
    }
    // [(frames), h, w, C] tokens -> [(frames), C, h, w]: egress with B = frames, F = 1
    if (egress_latent(t.p, t.ld, dst, 0, static_cast<int>(frames), t.C, 1, h, w, stream) != 0) return -3;
    return n;
}

}  // extern "C"
