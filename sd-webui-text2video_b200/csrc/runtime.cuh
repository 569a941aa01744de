// Host runtime shared by every network of the library (UNet, VAE decoder and encoder, text towers, adapter): parameter
// store, packed-weight cache, a lifetime-aware activation arena, the "plan" -- a flat list of pre-encoded kernel launches
// (tensor maps encoded once per shape) that one forward replays on a stream without any host-side shape logic -- and the
// per-handle cache of those plans.
#pragma once
#include "common.cuh"
#include "gemm_tc.cuh"
#include "kernels.cuh"
#include "shard.cuh"

#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <functional>
#include <list>
#include <map>
#include <memory>
#include <set>
#include <string>
#include <vector>

namespace t2v {

// ----------------------------------------------------------------------------------------- parameters
struct Param {
    std::vector<long long> shape;
    __half* data = nullptr;      // fp16 copy in the ORIGINAL (PyTorch) layout, library-owned (the EFFECTIVE weight: base + merged LoRAs)
    __half* base = nullptr;      // copy of the shipped weight, kept from the first LoRA merge on (lora_clear restores it bit for bit)
    long long elems = 0;
    bool expected = false;
    bool set = false;
};

// How one packed variant is (re)built from its sources: replayed in creation order when a source changes WITHOUT a new
// weights version (LoRA hot-merge), so packed buffers keep their addresses and every plan / captured graph stays valid.
struct PackRecipe {
    std::string key;
    std::vector<std::string> sources;      // parameter names and / or keys of other packed variants
    std::function<int(cudaStream_t)> run;
};

class ParamStore {
public:
    ~ParamStore();
    void expect(const std::string& name, std::vector<long long> shape);
    int set(const std::string& name, const void* src, int dtype, int ndim, const int64_t* shape, cudaStream_t s);
    int missing(std::string* one) const;
    bool complete(const char* what) const;      // false, with "<what> parameters missing (e.g. '<name>')" set, until all are set
    int info(int index, std::string* name, std::vector<long long>* shape) const;   // returns count, -1 if out of range
    const Param& get(const std::string& name) const;     // aborts via set_error + null data if absent
    bool has(const std::string& name) const { return params_.count(name) != 0; }
    // packed variants, created lazily and cached until any parameter changes
    __half* packed(const std::string& key) const;
    __half* new_packed(const std::string& key, long long elems);
    void invalidate_packed();
    unsigned long long version() const { return version_; }
    // packed-variant recipes (see PackRecipe) and the name a device pointer is known under ("" if unknown)
    void add_recipe(const std::string& key, std::vector<std::string> sources, std::function<int(cudaStream_t)> run);
    std::string key_of(const void* p) const;
    // LoRA hot-merge (stable_lora/stable_utils/lora_processor.py:50-96): data = fp16(data + fp16(fp16(B @ A) * alpha)), then only
    // the packed variants that depend on `name` are rebuilt in place.  temporal_mean: Conv3d (3,1,1) weights, the product is
    // viewed [out, in, 3, 3, 1] and averaged over the second kernel axis (:86-94).
    int lora_merge(const std::string& name, const __half* lora_A, const __half* lora_B, int rank, float alpha, int temporal_mean,
                   cudaStream_t s);
    // VideoCrafter LoRA (videocrafter/lvdm/models/modules/lora.py:620-672): data = fp16(data + alpha * up @ down) with fp32
    // factors / accumulation and one rounding (up [out, rank], down [rank, cols], dtype 0 fp16 / 1 fp32), then the same in-place
    // re-pack as lora_merge.  A removal (`-=`) is alpha negated.
    int lora_apply(const std::string& name, const void* up, const void* down, int dtype, int rank, float alpha, cudaStream_t s);
    // ONE merged weight back to its base copy (net_load_lora_v2's origin_weight restore, :727-736), base copy freed; a weight
    // carrying no merge is left as it is
    int lora_restore(const std::string& name, cudaStream_t s);
    int lora_clear(cudaStream_t s);          // every merged weight back to its base copy (bit-identical to never merging)
    int merged_count() const;

private:
    int repack(const std::vector<std::string>& dirty, cudaStream_t s);
    Param* mergeable(const char* what, const std::string& name, int rank, cudaStream_t s);   // loaded matrix / conv weight, base kept
    std::map<std::string, Param> params_;
    std::map<std::string, __half*> packed_;
    std::vector<PackRecipe> recipes_;
    unsigned long long version_ = 0;
};

// The C out-parameters of the handles' *_param_info / *_missing_params entry points.  param_info_out copies parameter
// `index` of `P` (name, ndim, up to 8 dims) and returns P's count, -1 if out of range; missing_params_out copies the name
// of one missing parameter and returns how many are missing.
int param_info_out(const ParamStore& P, int index, char* name_out, size_t name_cap, int64_t* shape_out, int* ndim_out);
int missing_params_out(const ParamStore& P, char* name_out, size_t name_cap);

// ----------------------------------------------------------------------------------------- arena
// Offsets are handed out by a first-fit free list while the plan is being built (the build order IS the execution
// order, so build-time lifetimes are run-time lifetimes).  A dry pass measures the peak, then the real pass runs
// against one cudaMalloc'ed slab.
class Arena {
public:
    void reset(char* base, bool no_reuse);
    char* alloc(size_t bytes);
    void free(char* p);
    size_t peak() const { return peak_; }
    long count() const { return count_; }

private:
    struct Blk { size_t off, size; };
    char* base_ = nullptr;
    bool no_reuse_ = false;
    long count_ = 0, limit_ = -1;
    size_t top_ = 0, peak_ = 0;
    std::vector<Blk> free_;
    std::map<size_t, size_t> live_;
};

struct Tok {                      // channels-last token matrix view
    __half* p = nullptr;
    long long rows = 0;
    int C = 0;
    long long ld = 0;
};

using Step = std::function<int(cudaStream_t)>;
enum StepKind : int { STEP_GEMM = 0, STEP_ATTN = 1, STEP_NORM = 2, STEP_OTHER = 3, STEP_NKINDS = 4 };
struct StepRec {
    Step fn;
    int kind;
    double flops;
    std::string label;
};

// Frame-sharded plans (shard.cuh): host-side state the exchange steps read at LAUNCH time -- the peers' mapped slabs and
// the byte offset of every exchange's destination buffer inside each peer's slab are only known after the ranks have
// swapped their exports (t2v_unet_shard_connect), which happens after the plan is built and before its first replay.
struct PlanShard {
    int fb[SHARD_MAX_RANKS + 1] = {0};                 // frame partition of the clip
    int n_xchg = 0, n_gn = 0;
    long long dst_off[SHARD_MAX_XCHG] = {0};           // this rank's destination offsets (bytes into its slab)
    long long peer_dst_off[SHARD_MAX_RANKS][SHARD_MAX_XCHG] = {{0}};
    char* peer_slab[SHARD_MAX_RANKS] = {nullptr};      // peer_slab[rank] = own slab
    bool connected = false;
    int own_rank = 0;
    ~PlanShard();
};

struct Plan {
    std::vector<StepRec> steps;
    std::shared_ptr<PlanShard> shard;
    char* slab = nullptr;
    size_t slab_bytes = 0;
    double flops = 0.0;
    int launches = 0;
    unsigned long long weights_version = 0;
    std::map<std::string, std::pair<Tok, std::pair<int, int>>> taps;    // name -> (tokens, (h, w))
    cudaGraphExec_t graph = nullptr;
    int eager_runs = 0;
    ~Plan();
};

// Helper that records launches into a plan (or only simulates allocations when `dry`).
class Builder {
public:
    Builder(Plan* plan, Arena* arena, bool dry, int sms) : plan_(plan), arena_(arena), dry_(dry), sms_(sms) {}
    bool dry() const { return dry_; }
    Tok alloc(long long rows, int C, int ld = 0);
    void* alloc_bytes(size_t bytes);
    void free(const Tok& t) { arena_->free(reinterpret_cast<char*>(t.p)); }
    void free_bytes(void* p) { arena_->free(reinterpret_cast<char*>(p)); }
    int gemm(GemmProblem& p);                                     // plans + records; returns 0 or <0
    void step(Step s, int launches = 1, int kind = STEP_OTHER, double flops = 0.0, const char* label = "");
    void add_flops(double f) { plan_->flops += f; }
    int sms() const { return sms_; }
    int error = 0;

private:
    Plan* plan_;
    Arena* arena_;
    bool dry_;
    int sms_;
};

// ----------------------------------------------------------------------------------------- layer helpers
struct NetCtx {
    ParamStore* params;
    Builder* b;
    cudaStream_t stream;      // weight-packing kernels are enqueued here while the plan is built
    void* gn_ws;              // zero-initialised groupnorm workspace (partials, stats, counters)
    const ShardPeers* shard_peers = nullptr;   // frame-sharded clip: live peer table (filled by connect), else null
    PlanShard* plan_shard = nullptr;
};
int round_up(int v, int m);
// packed-weight accessors (created on first use, cached in the ParamStore until a parameter changes)
const __half* w_conv(NetCtx& c, const std::string& name, int taps, int n_alloc = 0, int k_alloc = 0);
const __half* w_conv_kmajor(NetCtx& c, const std::string& name);
const __half* w_cat(NetCtx& c, const std::vector<std::string>& names);
struct Geglu { const __half* w; const __half* b; int bn; };
Geglu w_geglu(NetCtx& c, const std::string& prefix, int H, int K, int bn);
const __half* prm(NetCtx& c, const std::string& name);
// recorded ops
GemmProblem base_problem(const Tok& a, int K, const __half* w, int n_alloc, int N, const Tok& out);
Tok linear(NetCtx& c, const Tok& x, const __half* w, int N, const __half* bias, const Tok* residual, int K = 0);
// shard_total_rows > 0: 5-D norm of a pixel-sharded clip -- the statistics span `shard_total_rows` rows per sample over all ranks
Tok group_norm(NetCtx& c, const Tok& x, const std::string& prefix, long long rows_per_inst, float eps, bool silu,
               long long shard_total_rows = 0);
Tok layer_norm(NetCtx& c, const Tok& x, const std::string& prefix);
// y = Linear(LayerNorm(x)) (+residual) with the normalisation folded into the GEMM: a row-statistics kernel (reads x once)
// + one GEMM on the RAW rows whose epilogue applies rstd * (acc - mean * colsum) + bias'.  `w_src` [N, K] / `bias_src` are
// the (already concatenated / GEGLU-interleaved) weights; the gamma/beta-folded copy is cached under `key`.
Tok ln_linear(NetCtx& c, const Tok& x, const std::string& ln_prefix, const std::string& key, const __half* w_src,
              const __half* bias_src, int N, const Tok* residual, int flags = 0, int force_bn = 0);
Tok conv3x3(NetCtx& c, const Tok& x, const std::string& wname, const __half* bias, int bias_rows, long long bias_stride,
            int N, int hcur, int wcur, const Tok* residual, int n_alloc = 0);

// Runs the plan once with a CUDA-event pair around every step; out[kind*3 + {0,1,2}] = {ms, flops, launches}, out[12] = total ms.
// If T2V_PROFILE_DUMP names a file, one line per launch (index, kind, ms, flop, label) is written there.
int profile_plan(Plan* plan, cudaStream_t stream, double* out13);
// Replays the plan on `stream`.  The first call runs launch by launch; the second call captures the launch list into a
// CUDA graph (through a private capture stream: the caller's may be the legacy default stream) and from then on a
// forward is ONE cudaGraphLaunch -- the ~1k launches stop costing host time.  T2V_NO_GRAPH=1 disables it.
int run_plan(Plan* plan, cudaStream_t stream, bool allow_graph);

// ----------------------------------------------------------------------------------------- plan building and caching
// A network's plan builder: records (or, when `dry`, only counts) its launches into the plan, allocating from the arena.
using BuildFn = std::function<int(Plan* plan, Arena* arena, bool dry)>;

// The dry pass alone, on a scratch plan sharing `shard`: returns the peak activation bytes (-1 if the build failed) and
// stores the plan's algorithmic flop count in *flops.
long long dry_build(const std::shared_ptr<PlanShard>& shard, bool no_reuse, const BuildFn& build, double* flops = nullptr);
// The slab build_plan allocates for a dry-pass peak of `peak` bytes.
inline size_t plan_slab_bytes(long long peak) { return static_cast<size_t>(peak) + (1 << 20); }
// Builds `plan` (a shell: the caller may have set its shard): the dry pass measures the peak, one slab of peak + 1 MB is
// allocated, the real pass records the launches against it, and the plan is stamped with `weights_version`.  `label`
// names the network in the error message of a failed slab allocation.  Returns 0, or < 0 with the error set.
int build_plan(Plan* plan, unsigned long long weights_version, bool no_reuse, const char* label, const BuildFn& build);

// One handle's plans, each with its I/O staging record (where the inputs and outputs sit inside the plan's slab), keyed by
// shape and built for one weights version.  Every plan owns an activation slab (GBs at video shapes) and an instantiated
// graph, so at most `bound` are kept, evicting the least recently used.
template <class IO>
class PlanCache {
public:
    struct Entry {
        std::string key;
        std::unique_ptr<Plan> plan;
        IO io{};
    };
    explicit PlanCache(int bound) : bound_(static_cast<size_t>(std::max(bound, 1))) {}

    // The plan of `key` built for weights `version`, made the most recently used; null if there is none.
    Entry* find(const std::string& key, unsigned long long version) {
        for (auto it = entries_.begin(); it != entries_.end(); ++it)
            if (it->key == key && it->plan->weights_version == version) {
                entries_.splice(entries_.end(), entries_, it);
                return &entries_.back();
            }
        return nullptr;
    }
    // Whether the plan of `key` built for weights `version` is held, without touching the use order.
    bool holds(const std::string& key, unsigned long long version) const {
        return std::any_of(entries_.begin(), entries_.end(),
                           [&](const Entry& e) { return e.key == key && e.plan->weights_version == version; });
    }
    // Builds the plan of `key` from `shell` with build_plan, `fn(plan, arena, dry, &io)` filling the entry's I/O record, and
    // keeps it as the most recently used.  First drops every plan of an older weights version (versions only grow, so such
    // a plan can never be replayed again) and then the least recently used ones down to the bound.  Null on failure.
    template <class F>
    Entry* build(const std::string& key, unsigned long long version, cudaStream_t stream, std::unique_ptr<Plan> shell,
                 bool no_reuse, const char* label, F&& fn) {
        auto stale = [&](const Entry& e) { return e.plan->weights_version != version || e.key == key; };
        if (entries_.size() >= bound_ || std::any_of(entries_.begin(), entries_.end(), stale))
            cudaStreamSynchronize(stream);          // a plan about to be destroyed may still be in flight on this stream
        entries_.remove_if(stale);
        while (entries_.size() >= bound_) entries_.pop_front();
        Entry e{key, std::move(shell)};
        const int rc = build_plan(e.plan.get(), version, no_reuse, label,
                                  [&](Plan* p, Arena* a, bool dry) { return fn(p, a, dry, &e.io); });
        if (rc != 0) return nullptr;
        entries_.push_back(std::move(e));
        return &entries_.back();
    }
    Entry* latest() { return entries_.empty() ? nullptr : &entries_.back(); }      // the most recently used; null if none
    // Drops every plan (shard setup; a grown workspace that the plans captured by its old pointer).
    void clear(cudaStream_t stream) {
        if (entries_.empty()) return;
        cudaStreamSynchronize(stream);
        entries_.clear();
    }
    size_t size() const { return entries_.size(); }
    size_t slab_bytes() const {          // activation slabs of the cached plans, together
        size_t s = 0;
        for (const Entry& e : entries_) s += e.plan->slab_bytes;
        return s;
    }

private:
    size_t bound_;
    std::list<Entry> entries_;      // least recently used first
};

// The zero-initialised GroupNorm workspace (partials, statistics, counters) a handle's plans capture by pointer.
struct GnWorkspace {
    void* ptr = nullptr;
    size_t bytes = 0;
    ~GnWorkspace();
    // Grows the workspace to at least `need` bytes, zeroed on `stream`.  Returns true if the old pointer is gone (the
    // plans that captured it must be dropped); ptr is null if the allocation failed (error set).
    bool ensure(size_t need, cudaStream_t stream);
};

// conv taps helpers over row dims (w, h, frames) and (pixels, frames, samples)
void taps_3x3(GemmProblem& p);
void taps_temporal(GemmProblem& p);

}  // namespace t2v
