#include "runtime.cuh"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstdlib>
#include <cstring>

namespace t2v {

// ----------------------------------------------------------------------------------------- ParamStore
ParamStore::~ParamStore() {
    for (auto& kv : params_) {
        if (kv.second.data) cudaFree(kv.second.data);
        if (kv.second.base) cudaFree(kv.second.base);
    }
    invalidate_packed();
}

void ParamStore::add_recipe(const std::string& key, std::vector<std::string> sources, std::function<int(cudaStream_t)> run) {
    recipes_.push_back(PackRecipe{key, std::move(sources), std::move(run)});
}

std::string ParamStore::key_of(const void* p) const {
    if (p == nullptr) return "";
    for (auto& kv : params_)
        if (kv.second.data == p) return kv.first;
    for (auto& kv : packed_)
        if (kv.second == p) return kv.first;
    return "";
}

int ParamStore::repack(const std::vector<std::string>& dirty_in, cudaStream_t s) {
    std::set<std::string> dirty(dirty_in.begin(), dirty_in.end());
    for (auto& r : recipes_) {              // creation order = dependency order (a folded weight is created after its source pack)
        bool hit = false;
        for (auto& src : r.sources)
            if (dirty.count(src)) hit = true;
        if (!hit) continue;
        const int rc = r.run(s);
        if (rc != 0) {
            set_error("re-packing '%s' failed (%d)", r.key.c_str(), rc);
            return rc;
        }
        dirty.insert(r.key);
    }
    return 0;
}

Param* ParamStore::mergeable(const char* what, const std::string& name, int rank, cudaStream_t s) {
    auto it = params_.find(name);
    if (it == params_.end() || !it->second.set) {
        set_error("%s: parameter '%s' is not loaded", what, name.c_str());
        return nullptr;
    }
    Param& p = it->second;
    if (p.shape.size() < 2 || rank < 1) {
        set_error("%s: '%s' is not a matrix / conv weight", what, name.c_str());
        return nullptr;
    }
    if (p.base == nullptr) {
        const size_t bytes = ((p.elems + 7) / 8 * 8) * sizeof(__half);
        if (cudaMalloc(&p.base, bytes) != cudaSuccess) {
            set_error("%s: cudaMalloc of the base copy of '%s' failed", what, name.c_str());
            return nullptr;
        }
        if (cudaMemcpyAsync(p.base, p.data, bytes, cudaMemcpyDeviceToDevice, s) != cudaSuccess) {
            launch_status("LoRA base copy");
            return nullptr;
        }
    }
    return &p;
}

int ParamStore::lora_merge(const std::string& name, const __half* A, const __half* B, int rank, float alpha, int temporal_mean,
                           cudaStream_t s) {
    auto it = params_.find(name);
    if (temporal_mean && it != params_.end()) {
        const std::vector<long long>& sh = it->second.shape;
        if (!(sh.size() == 5 && sh[2] == 3 && sh[3] == 1 && sh[4] == 1)) {
            set_error("lora_merge: temporal_mean needs a Conv3d (3,1,1) weight, '%s' is not", name.c_str());
            return -2;
        }
    }
    Param* p = mergeable("lora_merge", name, rank, s);
    if (p == nullptr) return -1;
    const int out = static_cast<int>(p->shape[0]);
    const int cols = static_cast<int>(p->elems / out);
    int rc = lora_merge_weight(p->data, A, B, out, cols, rank, alpha, temporal_mean, s);
    if (rc != 0) return rc;
    return repack({name}, s);
}

int ParamStore::lora_apply(const std::string& name, const void* up, const void* down, int dtype, int rank, float alpha,
                           cudaStream_t s) {
    if (dtype != 0 && dtype != 1) {
        set_error("lora_apply('%s'): dtype must be 0 (fp16) or 1 (fp32)", name.c_str());
        return -3;
    }
    Param* p = mergeable("lora_apply", name, rank, s);
    if (p == nullptr) return -1;
    const int out = static_cast<int>(p->shape[0]);
    const int cols = static_cast<int>(p->elems / out);
    int rc = lora_apply_weight(p->data, up, down, dtype, out, cols, rank, alpha, s);
    if (rc != 0) return rc;
    return repack({name}, s);
}

int ParamStore::lora_restore(const std::string& name, cudaStream_t s) {
    auto it = params_.find(name);
    if (it == params_.end() || !it->second.expected) {
        set_error("lora_restore: no parameter '%s'", name.c_str());
        return -1;
    }
    Param& p = it->second;
    if (p.base == nullptr) return 0;
    if (cudaMemcpyAsync(p.data, p.base, ((p.elems + 7) / 8 * 8) * sizeof(__half), cudaMemcpyDeviceToDevice, s) != cudaSuccess)
        return launch_status("lora_restore copy");
    cudaStreamSynchronize(s);
    cudaFree(p.base);
    p.base = nullptr;
    return repack({name}, s);
}

int ParamStore::lora_clear(cudaStream_t s) {
    std::vector<std::string> dirty;
    for (auto& kv : params_) {
        Param& p = kv.second;
        if (p.base == nullptr) continue;
        cudaMemcpyAsync(p.data, p.base, ((p.elems + 7) / 8 * 8) * sizeof(__half), cudaMemcpyDeviceToDevice, s);
        cudaStreamSynchronize(s);
        cudaFree(p.base);
        p.base = nullptr;
        dirty.push_back(kv.first);
    }
    return dirty.empty() ? 0 : repack(dirty, s);
}

int ParamStore::merged_count() const {
    int n = 0;
    for (auto& kv : params_)
        if (kv.second.base != nullptr) ++n;
    return n;
}

void ParamStore::expect(const std::string& name, std::vector<long long> shape) {
    Param& p = params_[name];
    p.shape = std::move(shape);
    p.elems = 1;
    for (long long s : p.shape) p.elems *= s;
    p.expected = true;
}

int ParamStore::set(const std::string& name, const void* src, int dtype, int ndim, const int64_t* shape,
                    cudaStream_t s) {
    auto it = params_.find(name);
    if (it == params_.end() || !it->second.expected) {
        set_error("unexpected parameter '%s' (strict load, as load_state_dict(strict=True))", name.c_str());
        return -1;
    }
    Param& p = it->second;
    if (static_cast<int>(p.shape.size()) != ndim) {
        set_error("parameter '%s': rank %d, expected %d", name.c_str(), ndim, static_cast<int>(p.shape.size()));
        return -2;
    }
    for (int i = 0; i < ndim; ++i)
        if (p.shape[i] != shape[i]) {
            set_error("parameter '%s': dim %d is %lld, expected %lld", name.c_str(), i, static_cast<long long>(shape[i]),
                      p.shape[i]);
            return -2;
        }
    if (dtype != 0 && dtype != 1) {
        set_error("parameter '%s': dtype must be 0 (fp16) or 1 (fp32)", name.c_str());
        return -3;
    }
    if (!p.data) {
        // pad allocations to 16 B multiples so vector loads of tails stay in bounds
        if (cudaMalloc(&p.data, ((p.elems + 7) / 8 * 8) * sizeof(__half)) != cudaSuccess) {
            set_error("cudaMalloc failed for parameter '%s'", name.c_str());
            return -4;
        }
        cudaMemsetAsync(p.data, 0, ((p.elems + 7) / 8 * 8) * sizeof(__half), s);   // zero tail: padded bias reads
    }
    // fp16 sources (the normal case: the reference pipeline calls .half() on the model) are a plain device-to-device copy --
    // no kernel launch per parameter, so a process's launch list starts with the packing / forward kernels
    if (dtype == 0) {
        if (cudaMemcpyAsync(p.data, src, p.elems * sizeof(__half), cudaMemcpyDeviceToDevice, s) != cudaSuccess) {
            set_error("cudaMemcpyAsync failed for parameter '%s'", name.c_str());
            return -5;
        }
    } else {
        int rc = convert_to_f16(src, dtype, p.data, p.elems, s);
        if (rc != 0) return rc;
    }
    if (p.base != nullptr) {      // a re-shipped weight replaces base + merges alike
        cudaStreamSynchronize(s);
        cudaFree(p.base);
        p.base = nullptr;
    }
    p.set = true;
    ++version_;
    invalidate_packed();
    return 0;
}

int ParamStore::missing(std::string* one) const {
    int n = 0;
    for (auto& kv : params_)
        if (kv.second.expected && !kv.second.set) {
            if (n == 0 && one) *one = kv.first;
            ++n;
        }
    return n;
}

bool ParamStore::complete(const char* what) const {
    std::string miss;
    if (missing(&miss) == 0) return true;
    set_error("%s parameters missing (e.g. '%s')", what, miss.c_str());
    return false;
}

static void copy_name(const std::string& name, char* out, size_t cap) {
    if (out && cap > 0) {
        strncpy(out, name.c_str(), cap - 1);
        out[cap - 1] = 0;
    }
}

int param_info_out(const ParamStore& P, int index, char* name_out, size_t name_cap, int64_t* shape_out, int* ndim_out) {
    std::string name;
    std::vector<long long> shape;
    const int n = P.info(index, &name, &shape);
    if (n < 0) return -1;
    copy_name(name, name_out, name_cap);
    if (ndim_out) *ndim_out = static_cast<int>(shape.size());
    if (shape_out)
        for (size_t i = 0; i < shape.size() && i < 8; ++i) shape_out[i] = shape[i];
    return n;
}

int missing_params_out(const ParamStore& P, char* name_out, size_t name_cap) {
    std::string one;
    const int n = P.missing(&one);
    copy_name(one, name_out, name_cap);
    return n;
}

int ParamStore::info(int index, std::string* name, std::vector<long long>* shape) const {
    int i = 0, n = 0;
    bool found = false;
    for (auto& kv : params_) {
        if (!kv.second.expected) continue;
        if (i == index) {
            if (name) *name = kv.first;
            if (shape) *shape = kv.second.shape;
            found = true;
        }
        ++i;
        ++n;
    }
    return found ? n : -1;
}

const Param& ParamStore::get(const std::string& name) const {
    static Param empty;
    auto it = params_.find(name);
    if (it == params_.end() || !it->second.set) {
        set_error("parameter '%s' is not loaded", name.c_str());
        return empty;
    }
    return it->second;
}

__half* ParamStore::packed(const std::string& key) const {
    auto it = packed_.find(key);
    return it == packed_.end() ? nullptr : it->second;
}

__half* ParamStore::new_packed(const std::string& key, long long elems) {
    __half* p = nullptr;
    if (cudaMalloc(&p, ((elems + 7) / 8 * 8) * sizeof(__half)) != cudaSuccess) {
        set_error("cudaMalloc failed for packed weight '%s'", key.c_str());
        return nullptr;
    }
    packed_[key] = p;
    return p;
}

void ParamStore::invalidate_packed() {
    for (auto& kv : packed_) cudaFree(kv.second);
    packed_.clear();
    recipes_.clear();
}

// ----------------------------------------------------------------------------------------- Arena
void Arena::reset(char* base, bool no_reuse) {
    base_ = base;
    no_reuse_ = no_reuse;
    top_ = 0;
    peak_ = 0;
    free_.clear();
    live_.clear();
    count_ = 0;
    const char* lim = getenv("T2V_ARENA_REUSE_LIMIT");      // debugging aid: only the first N allocations may reuse freed blocks
    limit_ = lim ? atol(lim) : -1;
}

char* Arena::alloc(size_t bytes) {
    bytes = (bytes + 1023) & ~static_cast<size_t>(1023);
    if (bytes == 0) bytes = 1024;
    const long idx = count_++;
    if (getenv("T2V_ARENA_TRACE") && base_ != nullptr) fprintf(stderr, "[arena] alloc #%ld %zu bytes\n", idx, bytes);
    if (!no_reuse_ && (limit_ < 0 || idx < limit_)) {
        int best = -1;
        for (int i = 0; i < static_cast<int>(free_.size()); ++i)
            if (free_[i].size >= bytes && (best < 0 || free_[i].size < free_[best].size)) best = i;
        if (best >= 0) {
            const size_t off = free_[best].off;
            if (free_[best].size == bytes) free_.erase(free_.begin() + best);
            else {
                free_[best].off += bytes;
                free_[best].size -= bytes;
            }
            live_[off] = bytes;
            return base_ + off;
        }
    }
    const size_t off = top_;
    top_ += bytes;
    peak_ = std::max(peak_, top_);
    live_[off] = bytes;
    return base_ + off;
}

void Arena::free(char* p) {
    if (no_reuse_ || p == nullptr && base_ != nullptr) return;
    const size_t off = static_cast<size_t>(p - base_);
    auto it = live_.find(off);
    if (it == live_.end()) return;
    Blk b{off, it->second};
    live_.erase(it);
    // insert sorted + coalesce
    auto pos = std::lower_bound(free_.begin(), free_.end(), b, [](const Blk& a, const Blk& c) { return a.off < c.off; });
    pos = free_.insert(pos, b);
    const int i = static_cast<int>(pos - free_.begin());
    if (i + 1 < static_cast<int>(free_.size()) && free_[i].off + free_[i].size == free_[i + 1].off) {
        free_[i].size += free_[i + 1].size;
        free_.erase(free_.begin() + i + 1);
    }
    if (i > 0 && free_[i - 1].off + free_[i - 1].size == free_[i].off) {
        free_[i - 1].size += free_[i].size;
        free_.erase(free_.begin() + i);
    }
    // shrink the bump pointer when the tail is free
    if (!free_.empty() && free_.back().off + free_.back().size == top_) {
        top_ = free_.back().off;
        free_.pop_back();
    }
}

PlanShard::~PlanShard() {
    for (int r = 0; r < SHARD_MAX_RANKS; ++r)
        if (peer_slab[r] != nullptr && r != own_rank) cudaIpcCloseMemHandle(peer_slab[r]);
}

Plan::~Plan() {
    if (graph) cudaGraphExecDestroy(graph);
    if (slab) cudaFree(slab);
}

// ----------------------------------------------------------------------------------------- Builder
Tok Builder::alloc(long long rows, int C, int ld) {
    Tok t;
    t.rows = rows;
    t.C = C;
    t.ld = ld > 0 ? ld : C;
    t.p = reinterpret_cast<__half*>(arena_->alloc(static_cast<size_t>(rows) * t.ld * sizeof(__half)));
    return t;
}

void* Builder::alloc_bytes(size_t bytes) { return arena_->alloc(bytes); }

int Builder::gemm(GemmProblem& p) {
    double rows = 1;
    for (int d = 0; d < p.nd; ++d) rows *= p.dim[d];
    // Split-K for contractions whose output cannot fill the machine (low-resolution levels: rows = 768 / 3072 with K up to
    // 23040): each (tile, split) work item accumulates a K range into an fp32 partial, a fix-up kernel folds the partials
    // in a fixed order and applies bias / residual.  Deterministic; chosen only when >= half of the SMs would idle.
    if (p.splits <= 1 && gemm_splitk_unsupported(p) == nullptr) {
        const long long tiles_m = (static_cast<long long>(rows) + GEMM_BLOCK_M - 1) / GEMM_BLOCK_M;
        const long long tiles = tiles_m * ((p.N + 255) / 256);
        const int kt = p.ntaps * ((p.K + GEMM_BLOCK_K - 1) / GEMM_BLOCK_K);
        // the split count the kernel runs (no empty splits): the fix-up pass must not read partials nobody wrote
        const int S = gemm_split_count(
            p, static_cast<int>(std::min<long long>(std::min<long long>(sms_ / std::max<long long>(tiles, 1), kt / 4), 8)));
        // (64-wide tiles without split-K were measured equal within 0.3 % on the whole forward: same MMA time per CTA)
        if (tiles * 2 <= sms_ && S >= 2) {
            float* scratch = reinterpret_cast<float*>(arena_->alloc(static_cast<size_t>(gemm_splitk_scratch_elems(p, S)) * sizeof(float)));
            GemmProblem q = gemm_splitk_partials(p, S, scratch);
            q.force_bn = 256;
            const int rc = gemm(q);
            if (rc != 0) return rc;
            const GemmProblem o = p;
            step([=](cudaStream_t s) { return gemm_splitk_reduce(o, S, scratch, s); }, 1, STEP_OTHER, 0.0, "splitk_reduce");
            arena_->free(reinterpret_cast<char*>(scratch));
            return 0;
        }
    }
    plan_->flops += 2.0 * rows * p.N * p.K * p.ntaps;
    if (dry_) {
        plan_->launches += 1;
        return 0;
    }
    GemmPlan gp;
    int rc = gemm_plan(p, &gp, sms_);
    if (rc != 0) {
        set_error("gemm_plan failed (%d): rows %.0f N %d K %d taps %d", rc, rows, p.N, p.K, p.ntaps);
        error = rc;
        return rc;
    }
    char lab[192];
    snprintf(lab, sizeof(lab), "gemm rows=%.0f N=%d K=%d taps=%d bn=%d tiles=%dx%d grid=%d%s%s%s%s", rows, p.N, p.K, p.ntaps, gp.bn,
             gp.desc.tiles_m, gp.desc.tiles_n, gp.grid, (p.flags & GEMM_GEGLU) ? " geglu" : "", p.residual ? " +res" : "",
             gp.desc.splits > 1 ? " splitK" : "", gp.bs ? " Bstat" : "");
    plan_->steps.push_back(StepRec{[gp](cudaStream_t s) { return gemm_launch(gp, s); }, STEP_GEMM, gp.flops, lab});
    plan_->launches += 1;
    return 0;
}

void Builder::step(Step s, int launches, int kind, double flops, const char* label) {
    plan_->launches += launches;
    plan_->flops += flops;
    if (!dry_) plan_->steps.push_back(StepRec{std::move(s), kind, flops, label});
}

int profile_plan(Plan* plan, cudaStream_t stream, double* out13) {
    const size_t n = plan->steps.size();
    std::vector<cudaEvent_t> ev(n + 1);
    for (auto& e : ev) cudaEventCreate(&e);
    cudaEventRecord(ev[0], stream);
    int rc = 0;
    for (size_t i = 0; i < n && rc == 0; ++i) {
        rc = plan->steps[i].fn(stream);
        cudaEventRecord(ev[i + 1], stream);
    }
    cudaStreamSynchronize(stream);
    for (int i = 0; i < 13; ++i) out13[i] = 0.0;
    if (rc == 0) {
        FILE* f = nullptr;
        if (const char* path = getenv("T2V_PROFILE_DUMP")) f = fopen(path, "w");
        for (size_t i = 0; i < n; ++i) {
            float ms = 0.f;
            cudaEventElapsedTime(&ms, ev[i], ev[i + 1]);
            const int k = plan->steps[i].kind;
            out13[k * 3 + 0] += ms;
            out13[k * 3 + 1] += plan->steps[i].flops;
            out13[k * 3 + 2] += 1.0;
            out13[12] += ms;
            if (f) fprintf(f, "%zu\t%d\t%.4f\t%.4g\t%s\n", i, k, ms, plan->steps[i].flops, plan->steps[i].label.c_str());
        }
        if (f) fclose(f);
    }
    for (auto& e : ev) cudaEventDestroy(e);
    return rc;
}

int run_plan(Plan* plan, cudaStream_t stream, bool allow_graph) {
    static const bool graphs = getenv("T2V_NO_GRAPH") == nullptr;
    if (graphs && allow_graph) {
        if (plan->graph == nullptr && plan->eager_runs >= 1) {
            cudaStream_t cs = nullptr;
            if (cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking) == cudaSuccess) {
                if (cudaStreamBeginCapture(cs, cudaStreamCaptureModeRelaxed) == cudaSuccess) {
                    int rc = 0;
                    for (auto& s : plan->steps) {
                        rc = s.fn(cs);
                        if (rc != 0) break;
                    }
                    cudaGraph_t g = nullptr;
                    const cudaError_t e = cudaStreamEndCapture(cs, &g);
                    if (rc == 0 && e == cudaSuccess && g != nullptr) {
                        if (cudaGraphInstantiate(&plan->graph, g, 0) != cudaSuccess) plan->graph = nullptr;
                    }
                    if (g) cudaGraphDestroy(g);
                }
                cudaStreamDestroy(cs);
            }
            cudaGetLastError();
            if (plan->graph == nullptr) plan->eager_runs = -(1 << 30);      // capture failed: stay eager, do not retry
        }
        if (plan->graph != nullptr) return cudaGraphLaunch(plan->graph, stream) == cudaSuccess ? 0 : -20;
    }
    for (auto& s : plan->steps) {
        const int rc = s.fn(stream);
        if (rc != 0) return rc;
    }
    plan->eager_runs += 1;
    return 0;
}

long long dry_build(const std::shared_ptr<PlanShard>& shard, bool no_reuse, const BuildFn& build, double* flops) {
    Plan scratch;
    scratch.shard = shard;
    Arena arena;
    arena.reset(nullptr, no_reuse);
    if (build(&scratch, &arena, true) != 0) return -1;
    if (flops) *flops = scratch.flops;
    return static_cast<long long>(arena.peak());
}

int build_plan(Plan* plan, unsigned long long weights_version, bool no_reuse, const char* label, const BuildFn& build) {
    const long long peak = dry_build(plan->shard, no_reuse, build);
    if (peak < 0) return -1;
    const size_t bytes = plan_slab_bytes(peak);
    if (cudaMalloc(&plan->slab, bytes) != cudaSuccess) {
        plan->slab = nullptr;
        set_error("%s activation slab cudaMalloc(%zu MB) failed", label, bytes >> 20);
        return -1;
    }
    plan->slab_bytes = bytes;
    Arena arena;
    arena.reset(plan->slab, no_reuse);
    if (build(plan, &arena, false) != 0) return -1;
    plan->weights_version = weights_version;
    return 0;
}

GnWorkspace::~GnWorkspace() {
    if (ptr) cudaFree(ptr);
}

bool GnWorkspace::ensure(size_t need, cudaStream_t stream) {
    if (need <= bytes) return false;
    if (ptr) cudaFree(ptr);
    bytes = 0;
    if (cudaMalloc(&ptr, need) != cudaSuccess) {
        ptr = nullptr;
        set_error("groupnorm workspace cudaMalloc failed");
        return true;
    }
    cudaMemsetAsync(ptr, 0, need, stream);
    bytes = need;
    return true;
}

void taps_3x3(GemmProblem& p) {
    p.ntaps = 9;
    for (int ky = 0; ky < 3; ++ky)
        for (int kx = 0; kx < 3; ++kx) {
            const int t = ky * 3 + kx;
            p.tap_off[t][0] = kx - 1;
            p.tap_off[t][1] = ky - 1;
            p.tap_off[t][2] = 0;
            p.tap_off[t][3] = 0;
        }
}

void taps_temporal(GemmProblem& p) {
    p.ntaps = 3;
    for (int kt = 0; kt < 3; ++kt) {
        p.tap_off[kt][0] = 0;
        p.tap_off[kt][1] = kt - 1;
        p.tap_off[kt][2] = 0;
        p.tap_off[kt][3] = 0;
    }
}


// ----------------------------------------------------------------------------------------- shared layer helpers
int round_up(int v, int m) { return (v + m - 1) / m * m; }

// packed weights -------------------------------------------------------------------------------------------
// conv / linear weight [Cout, Cin, taps...] -> [taps][n_alloc][k_alloc]
const __half* w_conv(NetCtx& c, const std::string& name, int taps, int n_alloc, int k_alloc) {
    if (c.b->dry()) return nullptr;     // shape-only pass (flop / memory model): no parameters needed
    ParamStore& P = *c.params;
    const Param& prm = P.get(name);
    if (!prm.data) {
        c.b->error = -10;
        return nullptr;
    }
    const int cout = static_cast<int>(prm.shape[0]), cin = static_cast<int>(prm.shape[1]);
    if (n_alloc == 0) n_alloc = cout;
    if (k_alloc == 0) k_alloc = cin;
    if (taps == 1 && n_alloc == cout && k_alloc == cin) return prm.data;     // already [N][K]
    const std::string key = name + "#t" + std::to_string(taps) + "n" + std::to_string(n_alloc) + "k" + std::to_string(k_alloc);
    if (__half* p = P.packed(key)) return p;
    if (c.b->dry()) return nullptr;
    __half* dst = P.new_packed(key, static_cast<long long>(taps) * n_alloc * k_alloc);
    const __half* src = prm.data;
    auto recipe = [=](cudaStream_t s) { return pack_conv_weight(src, 0, dst, cout, cin, taps, n_alloc, k_alloc, s); };
    if (!dst || recipe(c.stream) != 0) c.b->error = -11;
    P.add_recipe(key, {name}, recipe);
    return dst;
}
// stride-2 conv weight [Cout, Cin, 3, 3] -> [1][Cout][9*Cin] with K index = tap*Cin + c (matches im2col_s2 columns)
const __half* w_conv_kmajor(NetCtx& c, const std::string& name) {
    if (c.b->dry()) return nullptr;
    ParamStore& P = *c.params;
    const Param& prm = P.get(name);
    if (!prm.data) {
        c.b->error = -10;
        return nullptr;
    }
    const int cout = static_cast<int>(prm.shape[0]), cin = static_cast<int>(prm.shape[1]);
    const std::string key = name + "#kmajor";
    if (__half* p = P.packed(key)) return p;
    if (c.b->dry()) return nullptr;
    // [9][Cout][Cin] first, then view-transpose by a second pack: treat as conv weight with "Cin" = 9*Cin, taps = 1
    // pack_conv_weight source index = (o*Cin + k)*taps + tap ; we want dst[o][tap*Cin + k] -> do it tap by tap
    __half* dst = P.new_packed(key, static_cast<long long>(cout) * 9 * cin);
    __half* tmp = P.new_packed(key + "#tmp", static_cast<long long>(9) * cout * cin);
    const __half* src = prm.data;
    auto recipe = [=](cudaStream_t s) {
        const int rc = pack_conv_weight(src, 0, tmp, cout, cin, 9, cout, cin, s);
        if (rc != 0) return rc;
        for (int tap = 0; tap < 9; ++tap)
            if (cudaMemcpy2DAsync(dst + static_cast<long long>(tap) * cin, static_cast<size_t>(9) * cin * 2,
                                  tmp + static_cast<long long>(tap) * cout * cin, static_cast<size_t>(cin) * 2,
                                  static_cast<size_t>(cin) * 2, cout, cudaMemcpyDeviceToDevice, s) != cudaSuccess)
                return launch_status("w_conv_kmajor copy");
        return 0;
    };
    if (!dst || !tmp || recipe(c.stream) != 0) {
        c.b->error = -11;
        return dst;
    }
    P.add_recipe(key, {name}, recipe);
    return dst;
}
// concatenated bias-free projections (q|k|v or k|v) -> one [sum N, K] matrix
const __half* w_cat(NetCtx& c, const std::vector<std::string>& names) {
    if (c.b->dry()) return nullptr;
    ParamStore& P = *c.params;
    std::string key = "cat";
    long long total = 0;
    for (auto& n : names) {
        key += "#" + n;
        const Param& prm = P.get(n);
        if (!prm.data) {
            c.b->error = -10;
            return nullptr;
        }
        total += prm.elems;
    }
    if (__half* p = P.packed(key)) return p;
    if (c.b->dry()) return nullptr;
    __half* dst = P.new_packed(key, total);
    if (!dst) {
        c.b->error = -11;
        return nullptr;
    }
    std::vector<std::pair<const __half*, long long>> parts;
    for (auto& n : names) {
        const Param& prm = P.get(n);
        parts.push_back({prm.data, prm.elems});
    }
    auto recipe = [=](cudaStream_t s) {
        long long off = 0;
        for (auto& pr : parts) {
            if (cudaMemcpyAsync(dst + off, pr.first, pr.second * sizeof(__half), cudaMemcpyDeviceToDevice, s) != cudaSuccess)
                return launch_status("w_cat copy");
            off += pr.second;
        }
        return 0;
    };
    recipe(c.stream);
    P.add_recipe(key, names, recipe);
    return dst;
}
Geglu w_geglu(NetCtx& c, const std::string& prefix, int H, int K, int bn) {
    if (c.b->dry()) return Geglu{nullptr, nullptr, bn};
    ParamStore& P = *c.params;
    const Param& w = P.get(prefix + ".weight");
    const Param& bb = P.get(prefix + ".bias");
    Geglu g{nullptr, nullptr, bn};
    if (!w.data || !bb.data) {
        c.b->error = -10;
        return g;
    }
    const std::string key = prefix + "#geglu" + std::to_string(bn);
    if (__half* p = P.packed(key)) {
        g.w = p;
        g.b = P.packed(key + "#b");
        return g;
    }
    if (c.b->dry()) return g;
    __half* wd = P.new_packed(key, static_cast<long long>(2) * H * K);
    __half* bd = P.new_packed(key + "#b", static_cast<long long>(2) * H);
    const __half* ws = w.data;
    const __half* bs = bb.data;
    auto recipe = [=](cudaStream_t s) { return pack_geglu_weight(ws, bs, 0, wd, bd, H, K, bn, s); };
    if (!wd || !bd || recipe(c.stream) != 0) c.b->error = -11;
    P.add_recipe(key, {prefix + ".weight", prefix + ".bias"}, recipe);
    P.add_recipe(key + "#b", {key}, [](cudaStream_t) { return 0; });       // the packed bias travels with the packed weight
    g.w = wd;
    g.b = bd;
    return g;
}
const __half* prm(NetCtx& c, const std::string& name) {
    if (c.b->dry()) return nullptr;
    const Param& p = (*c.params).get(name);
    if (!p.data) c.b->error = -10;
    return p.data;
}

// elementary ops -----------------------------------------------------------------------------------------------
GemmProblem base_problem(const Tok& a, int K, const __half* w, int n_alloc, int N, const Tok& out) {
    GemmProblem p;
    memset(&p, 0, sizeof(p));
    p.a = a.p;
    p.lda = a.ld;
    p.K = K;
    p.nd = 1;
    p.dim[0] = static_cast<int>(a.rows);
    p.ntaps = 1;
    p.b = w;
    p.n_alloc = n_alloc;
    p.N = N;
    p.b_batch_dim = -1;
    p.out = out.p;
    p.ldo = out.ld;
    p.alpha = 1.0f;
    return p;
}

// y = x W^T (+bias) (+residual)
Tok linear(NetCtx& c, const Tok& x, const __half* w, int N, const __half* bias, const Tok* residual, int K) {
    Tok y = c.b->alloc(x.rows, N);
    GemmProblem p = base_problem(x, K ? K : x.C, w, N, N, y);
    p.bias = bias;
    if (residual) {
        p.residual = residual->p;
        p.ldr = residual->ld;
    }
    c.b->gemm(p);
    return y;
}

Tok group_norm(NetCtx& c, const Tok& x, const std::string& prefix, long long rows_per_inst, float eps, bool silu,
               long long shard_total_rows) {
    Tok y = c.b->alloc(x.rows, x.C);
    const ShardPeers* peers = shard_total_rows > 0 ? c.shard_peers : nullptr;
    int slot = -1;
    if (peers != nullptr && c.plan_shard != nullptr) {
        slot = c.plan_shard->n_gn++;
        if (slot >= SHARD_MAX_GN) {
            set_error("frame-sharded plan: more than %d cross-rank GroupNorms", SHARD_MAX_GN);
            c.b->error = -30;
        }
    }
    const __half* g = prm(c, prefix + ".weight");
    const __half* bt = prm(c, prefix + ".bias");
    void* ws = c.gn_ws;
    const int sms = c.b->sms();
    const Tok xx = x;
    char lab[96];
    if (peers == nullptr) {
        // one launch: statistics -> per-instance barrier -> normalise(+SiLU) (norm.cu gn_fused_kernel; falls back to the two
        // kernels below inside groupnorm_silu when the grid cannot be co-resident)
        snprintf(lab, sizeof(lab), "gn_fused rows=%lld C=%d inst_rows=%lld", x.rows, x.C, rows_per_inst);
        c.b->step([=](cudaStream_t s) {
            return groupnorm_silu(xx.p, xx.ld, y.p, y.ld, xx.rows, xx.C, static_cast<int>(rows_per_inst), g, bt, eps, silu ? 1 : 0,
                                  ws, sms, s, 0);
        }, 1, STEP_NORM, 0.0, lab);
        return y;
    }
    snprintf(lab, sizeof(lab), "gn_stats rows=%lld C=%d inst_rows=%lld", x.rows, x.C, rows_per_inst);
    c.b->step([=](cudaStream_t s) {
        GnShard gs;
        memset(&gs, 0, sizeof(gs));
        gs.peers = *peers;          // read at launch: the peer table is filled by t2v_unet_shard_connect
        gs.slot = slot;
        gs.total_rows_per_inst = shard_total_rows;
        return groupnorm_silu(xx.p, xx.ld, y.p, y.ld, xx.rows, xx.C, static_cast<int>(rows_per_inst), g, bt, eps, silu ? 1 : 0,
                              ws, sms, s, 1, &gs);
    }, 1, STEP_NORM, 0.0, lab);
    snprintf(lab, sizeof(lab), "gn_apply rows=%lld C=%d inst_rows=%lld", x.rows, x.C, rows_per_inst);
    c.b->step([=](cudaStream_t s) {
        return groupnorm_silu(xx.p, xx.ld, y.p, y.ld, xx.rows, xx.C, static_cast<int>(rows_per_inst), g, bt, eps, silu ? 1 : 0,
                              ws, sms, s, 2);
    }, 1, STEP_NORM, 0.0, lab);
    return y;
}

Tok layer_norm(NetCtx& c, const Tok& x, const std::string& prefix) {
    Tok y = c.b->alloc(x.rows, x.C);
    const __half* g = prm(c, prefix + ".weight");
    const __half* bt = prm(c, prefix + ".bias");
    const Tok xx = x;
    char lab[96];
    snprintf(lab, sizeof(lab), "layernorm rows=%lld C=%d", x.rows, x.C);
    c.b->step([=](cudaStream_t s) { return layernorm(xx.p, xx.ld, y.p, y.ld, xx.rows, xx.C, g, bt, 1e-5f, s); }, 1, STEP_NORM, 0.0, lab);
    return y;
}


Tok ln_linear(NetCtx& c, const Tok& x, const std::string& ln_prefix, const std::string& key, const __half* w_src,
              const __half* bias_src, int N, const Tok* residual, int flags, int force_bn) {
    ParamStore& P = *c.params;
    const int K = x.C;
    const __half* wf = nullptr;
    const float* cs = nullptr;
    const float* b32 = nullptr;
    if (!c.b->dry()) {
        const std::string k = key + "#lnfold:" + ln_prefix;
        __half* w = P.packed(k);
        if (w == nullptr) {
            w = P.new_packed(k, static_cast<long long>(N) * K);
            __half* csh = P.new_packed(k + "#cs", 2LL * N);        // fp32 arrays live in the same cache (2 halves each)
            __half* bsh = P.new_packed(k + "#b32", 2LL * N);
            const __half* gam = prm(c, ln_prefix + ".weight");
            const __half* bet = prm(c, ln_prefix + ".bias");
            __half* wdst = w;
            auto recipe = [=](cudaStream_t s) {
                return fold_ln_into_linear(w_src, bias_src, gam, bet, wdst, reinterpret_cast<float*>(csh), reinterpret_cast<float*>(bsh),
                                           N, K, s);
            };
            if (!w || !csh || !bsh || recipe(c.stream) != 0) c.b->error = -12;
            P.add_recipe(k, {ln_prefix + ".weight", ln_prefix + ".bias", P.key_of(w_src), P.key_of(bias_src)}, recipe);
        }
        wf = w;
        cs = reinterpret_cast<const float*>(P.packed(k + "#cs"));
        b32 = reinterpret_cast<const float*>(P.packed(k + "#b32"));
    }
    float2* stats = reinterpret_cast<float2*>(c.b->alloc_bytes(static_cast<size_t>(x.rows) * sizeof(float2)));
    {
        const Tok xx = x;
        char lab[96];
        snprintf(lab, sizeof(lab), "ln_rowstats rows=%lld C=%d", x.rows, x.C);
        c.b->step([=](cudaStream_t s) { return layernorm_rowstats(xx.p, xx.ld, xx.rows, xx.C, 1e-5f, stats, s); }, 1, STEP_NORM,
                  0.0, lab);
    }
    const int ncols = (flags & GEMM_GEGLU) ? N / 2 : N;
    Tok y = c.b->alloc(x.rows, ncols);
    GemmProblem p = base_problem(x, K, wf, N, N, y);
    p.flags = flags | GEMM_LN;
    p.rowstat = stats;
    p.colsum = cs;
    p.bias32 = b32;
    p.force_bn = force_bn;
    if (residual) {
        p.residual = residual->p;
        p.ldr = residual->ld;
    }
    c.b->gemm(p);
    c.b->free_bytes(stats);
    return y;
}

Tok conv3x3(NetCtx& c, const Tok& x, const std::string& wname, const __half* bias, int bias_rows, long long bias_stride,
            int N, int hcur, int wcur, const Tok* residual, int n_alloc) {
    const int frames = static_cast<int>(x.rows / (static_cast<long long>(hcur) * wcur));
    const int k_alloc = x.C;       // activations may carry zero-padded channels (stem): weights padded to match
    const __half* w = w_conv(c, wname, 9, n_alloc ? n_alloc : N, k_alloc);
    Tok y = c.b->alloc(x.rows, N, N % 8 == 0 ? N : round_up(N, 8));
    GemmProblem p = base_problem(x, x.C, w, n_alloc ? n_alloc : N, N, y);
    p.nd = 3;
    p.dim[0] = wcur;
    p.dim[1] = hcur;
    p.dim[2] = frames;
    taps_3x3(p);
    p.bias = bias;
    p.bias_rows = bias_rows;
    p.bias_stride = bias_stride;
    if (residual) {
        p.residual = residual->p;
        p.ldr = residual->ld;
    }
    c.b->gemm(p);
    return y;
}


}  // namespace t2v
