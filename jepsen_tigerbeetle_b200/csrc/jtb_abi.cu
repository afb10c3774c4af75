// jtb_abi.cu — C ABI of libjtb_check.so (see include/jtb_check.h): context, device buffers,
// launchers.  There is no CPU fallback: every check runs its CUDA kernels or returns an error.
#include <algorithm>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <type_traits>
#include <vector>

#include "jtb_wgl.cuh"
#include "jtb_level.cuh"
#include "jtb_scout.cuh"
#include "jtb_scans.cuh"
#include "jtb_table_bench.cuh"
#include "jtb_partition.cuh"
#include "jtb_monotonic.cuh"
#include "jtb_counter_bounds.cuh"
#include "jtb_transfer_lookups.cuh"
#include "jtb_read_explanations.cuh"
#include "jtb_read_gaps.cuh"
#include "jtb_transfer_placement.cuh"
#include "jtb_serial_witness.cuh"
#include "jtb_repaired_witness.cuh"
#include "jtb_lifted_witness.cuh"
#include "jtb_class_witness.cuh"
#include "jtb_lookup_witness.cuh"
#include "jtb_witness.cuh"
#include "jtb_edn.cuh"
#include "jtb_edn_checks.cuh"
#include "jtb_set_edn.cuh"

using namespace jtb;

struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
};

struct jtb_ctx {
    int device = 0;
    jtb_opts opts{};
    cudaStream_t stream = nullptr;
    cudaStream_t scout_stream = nullptr;   // the depth-first scouts run beside the search kernel
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_setup = nullptr;
    int n_sms = 0;
    std::string err;
    std::mutex mu;  // a context serialises its calls; use one context per JVM thread for concurrency
    // cached device buffers (grown on demand, reused across calls)
    DevBuf table, pool, rows, classes, cls_inv, ctrl, found, maxrank;
    DevBuf sc_init, sc_tables, sc_stacks, sc_ctl;   // scouts: initial entries, private tables, stacks, control words
    SfBuffers sf;                        // set-full pass: its device buffers
    DevBuf lv_ctrl, lv_buf[2];          // level engine: control block, the two level arrays
    DevBuf lv_aux[2], lv_beam;          // beam mode: per-entry priority words, histogram + trackers
    size_t table_dirty = ~(size_t)0;    // bytes at the start of `table` that may hold old slots (level engine clears only these)
    int last_engine = 0;                // 0 work-list (visited table complete), 1 level (visited set is ephemeral)
    unsigned long long stats[24] = {0};
    unsigned long long last_configs = 0;  // configs of the previous search (sizes the next table)
    // what jtb_final_configs needs from the last search (its visited table is still in `table`)
    struct {
        bool valid = false;
        int64_t n_events = 0;
        int n_shards = 0, kw = 0;
        uint64_t n_slots = 0;
        std::vector<int> max_rank, verdict;
    } fc;
};

namespace {

double now_s() {
    return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

#define CK(call)                                                                             \
    do {                                                                                     \
        cudaError_t e_ = (call);                                                             \
        if (e_ != cudaSuccess) {                                                             \
            ctx->err = std::string(#call) + ": " + cudaGetErrorString(e_);                   \
            return -1;                                                                       \
        }                                                                                    \
    } while (0)

int ensure(jtb_ctx* ctx, DevBuf& b, size_t bytes) {
    if (bytes <= b.cap) return 0;
    if (b.p) CK(cudaFree(b.p));
    b.p = nullptr;
    b.cap = 0;
    size_t want = std::max<size_t>(bytes, 256);
    CK(cudaMalloc(&b.p, want));
    b.cap = want;
    return 0;
}

template <typename T>
int upload(jtb_ctx* ctx, DevBuf& b, const std::vector<T>& v) {
    ctx->stats[12] += v.size() * sizeof(T);  // host -> device bytes of this call
    if (ensure(ctx, b, v.size() * sizeof(T) + 64)) return -1;
    if (!v.empty()) CK(cudaMemcpyAsync(b.p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
    return 0;
}

// The one list of the (model, key width) combinations the search kernels are built for: bank and cas-register at 2, 4
// and 8 key words, set at 2 (register histories run the cas-register kernels).  Calls
// f(std::integral_constant<int, MODEL>, std::integral_constant<int, KW>).
template <typename F>
int dispatch_model_kw(jtb_ctx* ctx, int kind, int kw, F&& f) {
    using std::integral_constant;
    if (kind == JTB_MODEL_SET) return f(integral_constant<int, JTB_MODEL_SET>(), integral_constant<int, 2>());
    auto by_kw = [&](auto model) -> int {
        switch (kw) {
        case 2: return f(model, integral_constant<int, 2>());
        case 4: return f(model, integral_constant<int, 4>());
        case 8: return f(model, integral_constant<int, 8>());
        }
        ctx->err = "unsupported key width";
        return -1;
    };
    return kind == JTB_MODEL_BANK ? by_kw(integral_constant<int, JTB_MODEL_BANK>())
                                  : by_kw(integral_constant<int, JTB_MODEL_CAS_REGISTER>());
}

// two builds of the work-list kernel: Knossos-exact space (no eager-read code, 64 regs, JTB_CTAS_EXACT CTAs/SM) and the
// eager-read default (up to 80 regs, JTB_CTAS_EAGER CTAs/SM)
template <int MODEL, int KW>
int launch_wgl(jtb_ctx* ctx, const WglParams& p, int neg_ok, int grid, size_t smem) {
    auto k = p.eager_reads ? wgl_search_kernel<MODEL, KW, JTB_CTAS_EAGER, true> : wgl_search_kernel<MODEL, KW, JTB_CTAS_EXACT, false>;
    CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k<<<grid, WGL_THREADS, smem, ctx->stream>>>(p, neg_ok);
    CK(cudaGetLastError());
    return 0;
}

// the level engine (jtb_level.cuh): cooperative launch, every CTA resident (the levels are separated by grid barriers)
template <int MODEL, int KW>
int launch_level(jtb_ctx* ctx, const LvParams& p, int neg_ok, bool eager, int* grid_out) {
    constexpr int EW = KW + (MODEL == JTB_MODEL_BANK ? 4 : 0);
    const bool beam = p.beam_w != 0;
    const size_t smem = (beam ? sizeof(LvScratch<KW, EW, MODEL == JTB_MODEL_BANK, true>)
                              : sizeof(LvScratch<KW, EW, MODEL == JTB_MODEL_BANK, false>)) * LV_WARPS;
    const bool nk = !(MODEL == JTB_MODEL_BANK && !neg_ok);
    const void* k;
#define JTB_LVK(E, N, B) (const void*)level_search_kernel<MODEL, KW, E, (MODEL == JTB_MODEL_BANK ? N : true), B>
    if (beam) k = eager ? (nk ? JTB_LVK(true, true, true) : JTB_LVK(true, false, true)) : (nk ? JTB_LVK(false, true, true) : JTB_LVK(false, false, true));
    else k = eager ? (nk ? JTB_LVK(true, true, false) : JTB_LVK(true, false, false)) : (nk ? JTB_LVK(false, true, false) : JTB_LVK(false, false, false));
#undef JTB_LVK
    CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int per_sm = 0;
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, LV_THREADS, smem));
    if (per_sm < 1) { ctx->err = "level engine: the kernel does not fit on an SM"; return -1; }
    per_sm = std::min(per_sm, JTB_LV_CTAS);
    const int grid = ctx->opts.search_ctas ? std::min<int>((int)ctx->opts.search_ctas, ctx->n_sms * per_sm) : ctx->n_sms * per_sm;
    if (grid > 1024) { ctx->err = "level engine: more CTAs than barrier release words"; return -1; }
    *grid_out = grid;
    LvParams pp = p;
    void* args[] = {&pp};
    CK(cudaLaunchCooperativeKernel(k, dim3(grid), dim3(LV_THREADS), args, smem, ctx->stream));
    return 0;
}

// ---- level engine, host side: buffers, (re)launch, growth ------------------------------------------------------
// The search is ONE cooperative launch.  Only when a level outgrows the level arrays or the hash window does the kernel
// stop (cause TABLE_FULL) with the level it could not finish intact in its input array; the host then allocates 4x
// larger buffers, copies that one level over and relaunches from there.
// beam_w > 0: beam mode (jtb_level.cuh) — not exhaustive: only a VALID answer (shard_found) means anything.
int search_level(jtb_ctx* ctx, const jtb_model* m, const Prepared& P, int n_shards, const std::vector<int>& searchable,
                 const std::vector<uint64_t>& init_entries, Ctrl& hc, double& kernel_s, uint64_t& configs, uint64_t& probes,
                 uint32_t beam_w = 0) {
    const int KW = P.key_words;
    const bool bank = m->kind == JTB_MODEL_BANK;
    const int EW = KW + (bank ? 4 : 0);
    const bool eager = !(ctx->opts.flags & JTB_OPT_NO_EAGER_READS);
    size_t free_b = 0, total_b = 0;
    CK(cudaMemGetInfo(&free_b, &total_b));
    const size_t reserve = (size_t)4 << 30;
    const size_t avail = ctx->table.cap + ctx->lv_buf[0].cap + ctx->lv_buf[1].cap + (free_b > reserve ? free_b - reserve : 0);
    size_t table_bytes = ctx->opts.table_bytes ? ctx->opts.table_bytes
                         : (getenv("JTB_LV_TABLE_MB") ? (size_t)atoll(getenv("JTB_LV_TABLE_MB")) << 20 : (size_t)1 << 30);
    table_bytes = std::min(table_bytes, avail / 3);
    size_t buf_bytes = getenv("JTB_LV_BUF_MB") ? (size_t)atoll(getenv("JTB_LV_BUF_MB")) << 20 : (size_t)512 << 20;
    buf_bytes = std::max<size_t>(std::min(buf_bytes, avail / 3), init_entries.size() * 8 + 4096);
    auto slots_of = [&](size_t bytes) { uint64_t s = 1; while (s * 2 * KW * 8 <= bytes) s <<= 1; return s; };
    uint64_t table_slots = slots_of(std::max(table_bytes, ctx->table.cap));
    auto ensure_table = [&](uint64_t slots) -> int {
        const void* before = ctx->table.p;
        if (ensure(ctx, ctx->table, slots * KW * 8)) return -1;
        if (ctx->table.p != before) ctx->table_dirty = ~(size_t)0;
        return 0;
    };
    if (ensure_table(table_slots)) return -1;
    if (ensure(ctx, ctx->lv_buf[0], std::max(buf_bytes, ctx->lv_buf[0].cap)) || ensure(ctx, ctx->lv_buf[1], std::max(buf_bytes, ctx->lv_buf[1].cap)) ||
        ensure(ctx, ctx->lv_ctrl, sizeof(LvCtrl)))
        return -1;
    uint64_t buf_cap = std::min(ctx->lv_buf[0].cap, ctx->lv_buf[1].cap) / ((size_t)EW * 8);
    if (beam_w) {
        if (ensure(ctx, ctx->lv_aux[0], buf_cap * 4 + 64) || ensure(ctx, ctx->lv_aux[1], buf_cap * 4 + 64) ||
            ensure(ctx, ctx->lv_beam, sizeof(LvBeam)))
            return -1;
        std::vector<LvBeam> hb(1);
        std::memset(hb.data(), 0, sizeof(LvBeam));
        for (int k = 0; k < 3; ++k)
            for (int s = 0; s < LV_BEAM_SHARDS; ++s) { hb[0].min_crashed[k][s] = 0x7fffffff; hb[0].max_rank[k][s] = -1; }
        for (int s : searchable) { hb[0].min_crashed[0][s] = 0; hb[0].max_rank[0][s] = (int)P.rank_base[s]; }
        CK(cudaMemcpyAsync(ctx->lv_beam.p, hb.data(), sizeof(LvBeam), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemsetAsync(ctx->lv_aux[0].p, 0, init_entries.size() / EW * 4 + 64, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));   // `hb` must outlive the copy
    }
    // only what an earlier search may have written is cleared (the rest of the table is still zero)
    CK(cudaMemsetAsync(ctx->table.p, 0, std::min(ctx->table_dirty, (size_t)table_slots * KW * 8), ctx->stream));
    ctx->table_dirty = 0;
    LvCtrl lc;
    std::memset(&lc, 0, sizeof lc);
    lc.n_undecided = (int)searchable.size();
    CK(cudaMemcpyAsync(ctx->lv_ctrl.p, &lc, sizeof lc, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->lv_buf[0].p, init_entries.data(), init_entries.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
    LvParams p{};
    p.rows = (const int32_t*)ctx->rows.p;
    p.classes = (const ClassRec*)ctx->classes.p;
    p.cls_inv_pos = (const int32_t*)ctx->cls_inv.p;
    p.ctrl = (LvCtrl*)ctx->lv_ctrl.p;
    p.shard_found = (int*)ctx->found.p;
    p.shard_max_rank = (int*)ctx->maxrank.p;
    p.row_words = P.row_words;
    p.sum_off = P.sum_off;
    p.n_shards = n_shards;
    p.max_configs = ctx->opts.max_configs;
    p.time_budget_ns = (unsigned long long)ctx->opts.time_budget_ms * 1000000ull;
    p.narrow_max = getenv("JTB_LV_NARROW") ? (uint32_t)atoi(getenv("JTB_LV_NARROW")) : (uint32_t)(LV_WARPS * 8);
    p.slots_per_config = getenv("JTB_LV_SPC") ? (uint32_t)std::max(2, atoi(getenv("JTB_LV_SPC"))) : 16u;
    p.min_slots = 1ull << 16;
    std::memset(&p.init, 0, sizeof p.init);
    p.init.n_in = searchable.size();
    p.init.epoch = 1;
    p.init.s_in = 0; p.init.s_out = 1; p.init.s_spare = 2;
    p.init.contig = 1;
    p.init.beam_thr = -1;
    p.init.beam_frac = 1024;
    p.beam_w = beam_w;
    p.aux[0] = (uint32_t*)ctx->lv_aux[0].p;
    p.aux[1] = (uint32_t*)ctx->lv_aux[1].p;
    p.beam = (LvBeam*)ctx->lv_beam.p;
    p.init.win = 0;   // (set per launch below: needs the table size)
    CK(cudaEventRecord(ctx->ev0, ctx->stream));
    int attempts = 0, grid = 0;
    unsigned long long max_window = 0, max_width = 0, narrow_levels = 0, max_probe = 0;
    const double t_begin = now_s();
    for (;;) {
        ++attempts;
        p.table = (uint64_t*)ctx->table.p;
        p.table_slots = table_slots;
        p.min_slots = std::min<uint64_t>(p.min_slots, table_slots);
        p.buf[0] = (uint64_t*)ctx->lv_buf[0].p;
        p.buf[1] = (uint64_t*)ctx->lv_buf[1].p;
        p.buf_cap = buf_cap;
        p.seg_cap = buf_cap / LV_NSEG;
        p.init.zeroed = table_slots;
        p.init.win = lv_window(p, p.init.n_in, 0);
        if (ctx->opts.time_budget_ms) {   // what is left of the budget for this launch
            const double left = ctx->opts.time_budget_ms * 1e-3 - (now_s() - t_begin);
            p.time_budget_ns = (unsigned long long)(std::max(left, 1e-3) * 1e9);
        }
        const int neg_ok = bank ? m->negative_balances_ok : 0;
        if (int rc = dispatch_model_kw(ctx, m->kind, KW, [&](auto M, auto K) { return launch_level<M(), K()>(ctx, p, neg_ok, eager, &grid); }))
            return rc;
        CK(cudaMemcpyAsync(&lc, ctx->lv_ctrl.p, sizeof lc, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        if (lc.abort) { ctx->err = "level engine: a grid barrier timed out (internal error)"; return -1; }
#ifdef JTB_LV_PROF
        if (beam_w && getenv("JTB_BEAM_TRACE")) {
            for (int i = 0; i < 2048 && (i == 0 || lc.trace[i][1]); ++i)
                if (i < 40 || i % 25 == 0)
                    fprintf(stderr, "[beam W=%u] attempt %d level %d n_out %d thr %d frac %d min_c %d max_r %d\n", beam_w, i, lc.trace[i][0],
                            lc.trace[i][1], lc.trace[i][2], lc.trace[i][3], lc.trace[i][4], lc.trace[i][5]);
        }
        {
            const double wide = (double)std::max<unsigned long long>(lc.prof[9], 1), att = (double)std::max<unsigned long long>(lc.prof[8], 1);
            fprintf(stderr, "[lv prof] attempts %llu (wide %llu)  per attempt, cycles: phase1 %.0f phase2 %.0f flush %.0f | per wide level: "
                    "attempt %.0f barrier %.0f collect %.0f\n", lc.prof[8], lc.prof[9], lc.prof[0] / att, lc.prof[1] / att, lc.prof[2] / att,
                    lc.prof[3] / wide, lc.prof[4] / wide, lc.prof[5] / wide);
            unsigned long long bmin = ~0ull, bmax = 0, bsum = 0, wmin = ~0ull, wmax = 0, wsum = 0;
            for (int i = 0; i < grid; ++i) {
                bmin = std::min(bmin, lc.prof_cta[i][0]); bmax = std::max(bmax, lc.prof_cta[i][0]); bsum += lc.prof_cta[i][0];
                wmin = std::min(wmin, lc.prof_cta[i][1]); wmax = std::max(wmax, lc.prof_cta[i][1]); wsum += lc.prof_cta[i][1];
            }
            fprintf(stderr, "[lv prof] per CTA over the launch, Mcycles: busy min %.1f avg %.1f max %.1f | barrier wait min %.1f avg %.1f max %.1f\n",
                    bmin * 1e-6, bsum * 1e-6 / grid, bmax * 1e-6, wmin * 1e-6, wsum * 1e-6 / grid, wmax * 1e-6);
        }
#endif
        probes += lc.probes;
        max_window = std::max(max_window, lc.max_window);
        max_width = std::max(max_width, lc.max_width);
        max_probe = std::max(max_probe, lc.max_probe_len);
        narrow_levels += lc.narrow_levels;
        ctx->table_dirty = std::max(ctx->table_dirty, (size_t)std::max<uint64_t>(lc.max_window, p.min_slots) * KW * 8);
        if (!(lc.fin.stop == 2 && lc.fin.cause == JTB_CAUSE_TABLE_FULL)) break;
        if (beam_w) break;   // a beam that outgrows its arrays has failed as a beam: the caller falls back
        // ---- a level outgrew the arrays or the window: 4x of both, carry the unfinished level over -------------
        CK(cudaMemGetInfo(&free_b, &total_b));
        const size_t have = ctx->table.cap + ctx->lv_buf[0].cap + ctx->lv_buf[1].cap;
        const size_t room = have + (free_b > reserve ? free_b - reserve : 0);
        const size_t new_table = std::min<size_t>((size_t)table_slots * KW * 8 * 4, (size_t)64 << 30);
        const size_t new_buf = std::min(ctx->lv_buf[0].cap, ctx->lv_buf[1].cap) * 4;
        // peak while the unfinished level is copied over: its old array + the two new arrays + the new table
        if (new_table + 2 * new_buf + ctx->lv_buf[lc.fin.in_idx].cap > room) break;
        const int ii = lc.fin.in_idx;
        if (ctx->lv_buf[ii ^ 1].p) { CK(cudaFree(ctx->lv_buf[ii ^ 1].p)); ctx->lv_buf[ii ^ 1] = DevBuf(); }
        if (ctx->table.p) { CK(cudaFree(ctx->table.p)); ctx->table = DevBuf(); }
        DevBuf grown;
        if (ensure(ctx, grown, new_buf)) return -1;
        if (lc.fin.contig) {
            CK(cudaMemcpyAsync(grown.p, ctx->lv_buf[ii].p, (size_t)lc.fin.n_in * EW * 8, cudaMemcpyDeviceToDevice, ctx->stream));
        } else {   // gather the segments of the unfinished level into one contiguous run
            size_t off = 0;
            const size_t seg_cap = buf_cap / LV_NSEG;
            for (int sg = 0; sg < LV_NSEG; ++sg) {
                const size_t n = (size_t)lc.seg[lc.fin.s_in][sg].n;
                if (!n) continue;
                CK(cudaMemcpyAsync((char*)grown.p + off * EW * 8, (const char*)ctx->lv_buf[ii].p + (size_t)sg * seg_cap * EW * 8,
                                   n * EW * 8, cudaMemcpyDeviceToDevice, ctx->stream));
                off += n;
            }
            if (off != lc.fin.n_in) { ctx->err = "level engine: segment counts do not add up"; return -1; }
        }
        CK(cudaStreamSynchronize(ctx->stream));
        CK(cudaFree(ctx->lv_buf[ii].p));
        ctx->lv_buf[ii] = grown;
        if (ensure(ctx, ctx->lv_buf[ii ^ 1], new_buf)) return -1;
        table_slots = slots_of(new_table);
        if (ensure_table(table_slots)) return -1;
        CK(cudaMemsetAsync(ctx->table.p, 0, (size_t)table_slots * KW * 8, ctx->stream));
        ctx->table_dirty = 0;
        buf_cap = new_buf / ((size_t)EW * 8);
        // resume at the level that did not fit
        LvState r = lc.fin;
        r.stop = 0; r.cause = 0; r.boost = 0; r.attempt = 0; r.epoch = 1;
        r.s_in = 0; r.s_out = 1; r.s_spare = 2; r.contig = 1;
        p.init = r;
        const int undecided = lc.n_undecided;
        std::memset(&lc, 0, sizeof lc);
        lc.n_undecided = undecided;
        CK(cudaMemcpyAsync(ctx->lv_ctrl.p, &lc, sizeof lc, cudaMemcpyHostToDevice, ctx->stream));
    }
    CK(cudaEventRecord(ctx->ev1, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
    kernel_s = ms * 1e-3;
    configs = lc.fin.total;
    std::memset(&hc, 0, sizeof hc);
    hc.stop = lc.fin.stop;
    hc.cause = lc.fin.cause;
    hc.configs = lc.fin.total;
    hc.probes = probes;
    hc.n_undecided = lc.n_undecided;
    unsigned long long* st = ctx->stats;
    st[0] = configs; st[1] = probes; st[2] = lc.fin.level + 1; st[3] = max_width; st[4] = narrow_levels; st[5] = 0;
    st[6] = max_probe; st[7] = max_window; st[8] = (unsigned long long)grid; st[9] = buf_cap;
    st[10] = (unsigned long long)attempts; st[11] = (unsigned long long)(ms * 1e3);
    st[12] += init_entries.size() * 8 + sizeof(LvCtrl) + (size_t)n_shards * 4;
    st[13] = (unsigned long long)attempts * sizeof(LvCtrl) + (size_t)n_shards * 8;
    st[14] = (unsigned long long)attempts;
    st[19] = 1;   // engine: level
    return 0;
}

// Stops the scouts on every way out of a search (they only end on their own when their budget is spent).
struct ScoutGuard {
    jtb_ctx* ctx;
    bool active = false;
    explicit ScoutGuard(jtb_ctx* c) : ctx(c) {}
    int stop() {
        if (!active) return 0;
        active = false;
        static const unsigned long long one = 1;
        // an 8-byte pageable copy is staged at once; ctx->stream never waits for the scout stream
        cudaError_t e = cudaMemcpyAsync((unsigned long long*)ctx->sc_ctl.p + 1, &one, 8, cudaMemcpyHostToDevice, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->scout_stream);
        if (e != cudaSuccess) { ctx->err = std::string("stopping the scouts: ") + cudaGetErrorString(e); return -1; }
        return 0;
    }
    ~ScoutGuard() { stop(); }
};

// CUDA loads kernels lazily, and loading one synchronizes the context: the first launch of a search / compact /
// re-hash kernel would wait for the running scouts (for seconds).  So every kernel
// a search can need is loaded before the scouts start.
template <typename K>
int preload(jtb_ctx* ctx, K kernel) {
    cudaFuncAttributes a;
    CK(cudaFuncGetAttributes(&a, kernel));
    return 0;
}

template <int MODEL, int KW>
int preload_search(jtb_ctx* ctx, bool eager) {
    constexpr int EW = KW + (MODEL == JTB_MODEL_BANK ? 4 : 0);
    int rc = eager ? (preload(ctx, wgl_search_kernel<MODEL, KW, JTB_CTAS_EAGER, true>) | preload(ctx, wgl_scout_kernel<MODEL, KW, true>))
                   : (preload(ctx, wgl_search_kernel<MODEL, KW, JTB_CTAS_EXACT, false>) | preload(ctx, wgl_scout_kernel<MODEL, KW, false>));
    rc |= preload(ctx, table_rehash_kernel<KW>) | preload(ctx, ring_compact_kernel<EW>) | preload(ctx, wgl_resume_ctrl_kernel);
    return rc ? -1 : 0;
}

template <int MODEL, int KW>
int launch_scout(jtb_ctx* ctx, const WglParams& p, const ScoutParams& sp, int neg_ok, int n_scouts) {
    if (p.eager_reads) wgl_scout_kernel<MODEL, KW, true><<<n_scouts, 32, 0, ctx->scout_stream>>>(p, sp, neg_ok);
    else wgl_scout_kernel<MODEL, KW, false><<<n_scouts, 32, 0, ctx->scout_stream>>>(p, sp, neg_ok);
    CK(cudaGetLastError());
    return 0;
}

// What one search leaves for the verdicts.
struct Search {
    Ctrl hc;                            // stop / cause / overflow
    std::vector<int> found, max_rank;   // per shard: found VALID, furthest frontier rank reached
    double kernel_s = 0;
    uint64_t configs = 0, probes = 0;
    uint64_t n_slots = 0;               // work list: slots of the visited table (jtb_final_configs reads it)
    explicit Search(int n_shards) : found(n_shards, 0), max_rank(n_shards, 0) { std::memset(&hc, 0, sizeof hc); }
};

// Per-shard results on the device before a search: nothing found, furthest rank = the shard's first rank.
int arm_shards(jtb_ctx* ctx, const Prepared& P, int n_shards, std::vector<int>& max_rank) {
    CK(cudaMemsetAsync(ctx->found.p, 0, n_shards * sizeof(int), ctx->stream));
    for (int s = 0; s < n_shards; ++s) max_rank[s] = (int)P.rank_base[s];
    CK(cudaMemcpyAsync(ctx->maxrank.p, max_rank.data(), n_shards * sizeof(int), cudaMemcpyHostToDevice, ctx->stream));
    return 0;
}

// ---- work-list engine, host side: ring and visited table, scouts, pause / grow / resume ------------------------
// The persistent kernel pauses when its ring or its table is nearly full; the host then compacts the live ring entries
// into a 4x larger ring and/or re-hashes the table into a 4x larger one and relaunches, so no work is lost.
// max_configs: stop (UNKNOWN) after this many configurations, 0 = no budget; scouts: run the depth-first scouts beside
// the search on histories with crashed ops.  t_start: start of the call (the scouts' grace period ends with its time budget).
int search_worklist(jtb_ctx* ctx, const jtb_history* h, const jtb_model* m, const Prepared& P,
                    const std::vector<int>& searchable, const std::vector<uint64_t>& init_entries, uint64_t max_configs,
                    bool scouts_on, double t_start, Search& r) {
    const int n_shards = h->n_shards;
    const int KW = P.key_words;
    const int EW = KW + (m->kind == JTB_MODEL_BANK ? 4 : 0);
    const int neg_ok = m->kind == JTB_MODEL_BANK ? m->negative_balances_ok : 0;
    const bool eager_mode = !(ctx->opts.flags & JTB_OPT_NO_EAGER_READS);
    Ctrl& hc = r.hc;
    ctx->last_engine = 0;
    ctx->table_dirty = ~(size_t)0;   // the work-list engine fills the table
    // CTA deque / grid: one WARP per configuration (jtb_wgl.cuh), every child of a configuration probed in the same
    // round trip
    const int cand_rounds = P.S_pad / 32, cls_rounds = (P.max_nc + 31) / 32;
    // worst case of children one CTA step can push (overflow -> ring)
    const uint32_t worst_push = (WGL_BATCH + WGL_WARPS) * 32 * (cand_rounds + cls_rounds);
    uint32_t deque_cap = 1024;                       // fixed: a full deque overflows to the ring
    while ((size_t)deque_cap * EW * 8 > 48 * 1024) deque_cap >>= 1;
    const uint32_t stage_cap = std::max(deque_cap, worst_push);
    const size_t smem = (size_t)(deque_cap + WGL_BATCH) * EW * 8;
    // eager-read searches are small and latency-bound: 3 CTAs/SM (no register spills) wins; the Knossos-exact space is
    // throughput-bound: 4 CTAs/SM (measured A/B, DESIGN.md)
    const int want_ctas = eager_mode ? JTB_CTAS_EAGER : JTB_CTAS_EXACT;
    const int ctas_per_sm = std::max(1, (int)std::min<size_t>(want_ctas, (220 * 1024) / (smem + 1024)));
    const int grid = ctx->opts.search_ctas ? (int)ctx->opts.search_ctas : ctx->n_sms * ctas_per_sm;
    const uint64_t per_step_push = (uint64_t)grid * stage_cap;  // worst case children of one step of every CTA
    // work ring
    uint64_t ring_entries = 1ull << 22;
    while (ring_entries < 4 * per_step_push + 2 * searchable.size()) ring_entries <<= 1;
    // test hook: start with a ring that is too small so that the RING_FULL pause/grow/resume path runs
    const bool tiny_ring = getenv("JTB_TEST_TINY_RING") != nullptr;
    if (ensure(ctx, ctx->pool, ring_entries * EW * 8)) return -1;
    CK(cudaMemsetAsync(ctx->pool.p, 0, ring_entries * EW * 8, ctx->stream));
    CK(cudaMemcpyAsync(ctx->pool.p, init_entries.data(), init_entries.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
    // visited table: start at 1 GiB (or the caller's size), grow x4 on load > 0.7 without losing work
    size_t free_b = 0, total_b = 0;
    CK(cudaMemGetInfo(&free_b, &total_b));
    const size_t reserve = (size_t)4 << 30;
    size_t max_table = ctx->opts.table_bytes ? ctx->opts.table_bytes : (size_t)64 << 30;
    max_table = std::min(max_table, ctx->table.cap + (free_b > reserve ? free_b - reserve : 0));
    // start at 1 GiB, or at 4x what the previous call on this context ended up needing (warm context)
    const size_t min_start = getenv("JTB_TABLE_START_MB") ? (size_t)atoll(getenv("JTB_TABLE_START_MB")) << 20 : (size_t)1 << 30;
    size_t start_bytes = std::max<size_t>(min_start, (size_t)ctx->last_configs * 4 * KW * 8);
    size_t table_bytes = std::min<size_t>(max_table, ctx->opts.table_bytes ? ctx->opts.table_bytes : start_bytes);
    uint64_t n_slots = 1;
    while (n_slots * 2 * KW * 8 <= table_bytes) n_slots <<= 1;
    if (ensure(ctx, ctx->table, n_slots * KW * 8)) return -1;
    CK(cudaMemsetAsync(ctx->table.p, 0, n_slots * KW * 8, ctx->stream));
    hc.tail = searchable.size();
    hc.created = searchable.size();
    hc.n_undecided = (int)searchable.size();
    CK(cudaMemcpyAsync(ctx->ctrl.p, &hc, sizeof hc, cudaMemcpyHostToDevice, ctx->stream));
    if (arm_shards(ctx, P, n_shards, r.max_rank)) return -1;
    DevBuf ring2, table2;  // growth targets (freed below)
    // cudaFree synchronizes the whole device, i.e. it would wait for the scouts: while they run, frees are deferred
    // (cudaFree is valid for stream-ordered allocations too)
    ScoutGuard scouts(ctx);
    std::vector<void*> deferred;
    auto free_tmp = [&]() {
        scouts.stop();
        for (void* q : deferred) cudaFree(q);
        deferred.clear();
        if (ring2.p) cudaFree(ring2.p);
        if (table2.p) cudaFree(table2.p);
        ring2 = DevBuf(); table2 = DevBuf();
    };
    auto grow_buf = [&](DevBuf& b, size_t bytes) -> int {
        if (bytes <= b.cap) return 0;
        if (b.p) { if (scouts.active) deferred.push_back(b.p); else cudaFree(b.p); }
        b = DevBuf();
        // cudaMalloc also synchronizes with running kernels (the search would sit behind the scouts for seconds at
        // its first table growth); the stream-ordered allocator does not
        const cudaError_t e = scouts.active ? cudaMallocAsync(&b.p, bytes, ctx->stream) : cudaMalloc(&b.p, bytes);
        if (e != cudaSuccess) {
            (void)cudaGetLastError();
            b.p = nullptr;
            if (scouts.stop()) return -1;   // out of memory with frees pending: give the scouts up
            for (void* q : deferred) cudaFree(q);
            deferred.clear();
            CK(cudaMalloc(&b.p, bytes));
        }
        b.cap = bytes;
        return 0;
    };
    int attempts = 0;
    CK(cudaEventRecord(ctx->ev0, ctx->stream));
    WglParams pb{};   // what the search kernel and the scouts share
    pb.rows = (const int32_t*)ctx->rows.p;
    pb.classes = (const ClassRec*)ctx->classes.p;
    pb.cls_inv_pos = (const int32_t*)ctx->cls_inv.p;
    pb.ctrl = (Ctrl*)ctx->ctrl.p;
    pb.shard_found = (int*)ctx->found.p;
    pb.shard_max_rank = (int*)ctx->maxrank.p;
    pb.row_words = P.row_words;
    pb.S_pad = P.S_pad;
    pb.n_shards = n_shards;
    pb.max_nc = P.max_nc;
    pb.eager_reads = eager_mode ? 1 : 0;
    // ---- depth-first scouts (jtb_scout.cuh): only where the crowd is known to drown — histories with
    //      crashed ops — and launched FIRST so that they are resident before the persistent CTAs fill the SMs
    int64_t max_shard_events = 0;
    for (int s : searchable) max_shard_events = std::max<int64_t>(max_shard_events, h->shard_off[s + 1] - h->shard_off[s]);
    int n_scouts = 0;
    const bool scout_only = getenv("JTB_SCOUT_ONLY") != nullptr;   // test hook: no search kernel at all
    if (scouts_on && (P.max_nc > 0 || scout_only) && max_shard_events < (1ll << 29)) {
        n_scouts = getenv("JTB_SCOUTS") ? std::max(1, atoi(getenv("JTB_SCOUTS"))) : SCOUT_ORDERS;
        ScoutParams sp{};
        sp.n_init = (int)searchable.size();
        sp.n_orders = getenv("JTB_SCOUT_ORDERS") ? std::min(SCOUT_ORDERS, std::max(1, atoi(getenv("JTB_SCOUT_ORDERS")))) : SCOUT_ORDERS;
        const uint64_t sc_slots = 1ull << 22;                       // 2 M configs per scout
        sp.slot_mask = sc_slots - 1;
        sp.stack_cap = (uint32_t)(max_shard_events + 2);            // a path linearizes each op at most once
        sp.pair_budget = 8ull << 20;
        if (upload(ctx, ctx->sc_init, init_entries) ||
            ensure(ctx, ctx->sc_tables, (size_t)n_scouts * sc_slots * KW * 8) ||
            ensure(ctx, ctx->sc_stacks, (size_t)n_scouts * sp.stack_cap * (EW + 1) * 8) ||
            ensure(ctx, ctx->sc_ctl, SCOUT_CTL_WORDS * 8))
            return -1;
        CK(cudaMemsetAsync(ctx->sc_tables.p, 0, (size_t)n_scouts * sc_slots * KW * 8, ctx->stream));
        CK(cudaMemsetAsync(ctx->sc_ctl.p, 0, SCOUT_CTL_WORDS * 8, ctx->stream));
        sp.init = (const uint64_t*)ctx->sc_init.p;
        sp.tables = (uint64_t*)ctx->sc_tables.p;
        sp.stacks = (uint64_t*)ctx->sc_stacks.p;
        sp.ctl = (unsigned long long*)ctx->sc_ctl.p;
        CK(cudaEventRecord(ctx->ev_setup, ctx->stream));
        CK(cudaStreamWaitEvent(ctx->scout_stream, ctx->ev_setup, 0));
        if (int rc = dispatch_model_kw(ctx, m->kind, KW, [&](auto M, auto K) {
                return preload_search<M(), K()>(ctx, eager_mode) ? -1 : launch_scout<M(), K()>(ctx, pb, sp, neg_ok, n_scouts);
            }))
            return rc;
        scouts.active = true;
    }
    for (;;) {
        ++attempts;
        if (scout_only) { hc.stop = 2; hc.cause = JTB_CAUSE_BUDGET; break; }
        WglParams p = pb;
        p.table = (uint64_t*)ctx->table.p;
        p.slot_mask = n_slots - 1;
        p.ring = (uint64_t*)ctx->pool.p;
        p.ring_mask = ring_entries - 1;
        p.ring_guard = (tiny_ring && attempts == 1) ? 20000 : ring_entries - 3 * per_step_push;
        const uint64_t load_guard = (uint64_t)(0.50 * (double)n_slots);  // linear probing: keep chains short
        p.max_configs = load_guard;
        p.budget_cause = JTB_CAUSE_TABLE_FULL;
        if (max_configs && max_configs <= load_guard) {
            p.max_configs = max_configs;
            p.budget_cause = JTB_CAUSE_BUDGET;
        }
        p.time_budget_ns = (unsigned long long)ctx->opts.time_budget_ms * 1000000ull;
        p.deque_cap = deque_cap;
        if (int rc = dispatch_model_kw(ctx, m->kind, KW, [&](auto M, auto K) { return launch_wgl<M(), K()>(ctx, p, neg_ok, grid, smem); })) {
            free_tmp();
            return rc;
        }
        CK(cudaMemcpyAsync(&hc, ctx->ctrl.p, sizeof hc, cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        const bool grow_table = hc.stop == 2 && hc.cause == JTB_CAUSE_TABLE_FULL && n_slots * KW * 8 * 4 <= max_table;
        const bool grow_ring = hc.stop == 2 && hc.cause == CAUSE_RING_FULL && ring_entries * EW * 8 * 4 <= ((size_t)16 << 30);
        if (!grow_table && !grow_ring) break;
        if (hc.n_undecided <= 0) break;   // the scouts decided every shard while the search was pausing
        // ---- pause/resume: the live work is exactly the non-zero ring slots ---------------------
        const uint64_t new_ring_entries = grow_ring ? ring_entries * 4 : ring_entries;
        if (grow_buf(ring2, new_ring_entries * EW * 8)) {   // no memory for the larger ring: give up like a full table
            (void)cudaGetLastError();
            hc.stop = 2; hc.cause = JTB_CAUSE_TABLE_FULL;
            break;
        }
        CK(cudaMemsetAsync(ring2.p, 0, new_ring_entries * EW * 8, ctx->stream));
        Ctrl* dc = (Ctrl*)ctx->ctrl.p;
        CK(cudaMemsetAsync(&dc->tail, 0, sizeof(unsigned long long), ctx->stream));
        dispatch_model_kw(ctx, m->kind, KW, [&](auto M, auto K) {
            ring_compact_kernel<EntryLayout<M(), K()>::EW><<<ctx->n_sms * 8, 256, 0, ctx->stream>>>(
                (const uint64_t*)ctx->pool.p, ring_entries - 1, 0, ring_entries, (uint64_t*)ring2.p, new_ring_entries - 1, &dc->tail);
            return 0;
        });
        CK(cudaGetLastError());
        std::swap(ctx->pool, ring2);
        ring_entries = new_ring_entries;
        CK(cudaMemsetAsync(&dc->head, 0, sizeof(unsigned long long), ctx->stream));
        wgl_resume_ctrl_kernel<<<1, 1, 0, ctx->stream>>>(dc);   // stop, cause := 0 (unless everything is decided)
        CK(cudaGetLastError());
        if (grow_table) {
            const uint64_t new_slots = n_slots * 4;
            if (grow_buf(table2, new_slots * KW * 8)) {   // old + 4x table do not fit together: UNKNOWN, not an error
                (void)cudaGetLastError();
                hc.stop = 2; hc.cause = JTB_CAUSE_TABLE_FULL;
                break;
            }
            CK(cudaMemsetAsync(table2.p, 0, new_slots * KW * 8, ctx->stream));
            dispatch_model_kw(ctx, m->kind, KW, [&](auto, auto K) {
                table_rehash_kernel<K()><<<ctx->n_sms * 8, 256, 0, ctx->stream>>>((const uint64_t*)ctx->table.p, n_slots,
                                                                                  (uint64_t*)table2.p, new_slots - 1, &dc->overflow);
                return 0;
            });
            CK(cudaGetLastError());
            CK(cudaStreamSynchronize(ctx->stream));
            std::swap(ctx->table, table2);
            if (table2.p) {   // release the old table right away (deferred while the scouts run)
                if (scouts.active) deferred.push_back(table2.p); else cudaFree(table2.p);
                table2 = DevBuf();
            }
            n_slots = new_slots;
        }
    }
    unsigned long long sc_ctl[SCOUT_CTL_WORDS] = {0};
    if (n_scouts) {
        // the search gave up (UNKNOWN) while scouts are still walking: give them a grace period
        if (hc.stop == 2 && hc.n_undecided > 0) {
            double grace_s = getenv("JTB_SCOUT_GRACE_MS") ? atof(getenv("JTB_SCOUT_GRACE_MS")) * 1e-3 : 20.0;
            if (ctx->opts.time_budget_ms)
                grace_s = std::max(0.0, ctx->opts.time_budget_ms * 1e-3 - (now_s() - t_start));
            const double deadline = now_s() + grace_s;
            while (now_s() < deadline && cudaStreamQuery(ctx->scout_stream) == cudaErrorNotReady)
                std::this_thread::sleep_for(std::chrono::microseconds(200));
        }
        (void)cudaGetLastError();
        if (scouts.stop()) { free_tmp(); return -1; }
        CK(cudaMemcpyAsync(sc_ctl, ctx->sc_ctl.p, sizeof sc_ctl, cudaMemcpyDeviceToHost, ctx->stream));
    }
    CK(cudaEventRecord(ctx->ev1, ctx->stream));
    CK(cudaMemcpyAsync(r.found.data(), ctx->found.p, n_shards * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(r.max_rank.data(), ctx->maxrank.p, n_shards * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    free_tmp();
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1));
    r.kernel_s = ms * 1e-3;
    r.configs = hc.configs;
    r.probes = hc.probes;
    r.n_slots = n_slots;
    ctx->last_configs = hc.configs;
    unsigned long long* st = ctx->stats;
    st[0] = hc.configs; st[1] = hc.probes; st[2] = hc.expansions; st[3] = hc.tail;
    st[4] = hc.head; st[5] = hc.polls; st[6] = hc.max_probe_len; st[7] = n_slots;
    st[8] = (unsigned long long)grid; st[9] = ring_entries; st[10] = (unsigned long long)attempts;
    st[11] = (unsigned long long)(ms * 1e3);
    st[12] += init_entries.size() * 8 + sizeof(Ctrl) + (size_t)n_shards * 4;
    st[13] = (unsigned long long)attempts * sizeof(Ctrl) + (size_t)n_shards * 8;  // device -> host bytes
    st[14] = (unsigned long long)((scout_only ? 0 : attempts) + 3 * (attempts - 1) + (n_scouts ? 1 : 0));  // search + compact/rehash/re-arm + scouts
    st[15] = sc_ctl[2]; st[16] = sc_ctl[3]; st[17] = sc_ctl[4]; st[18] = (unsigned long long)n_scouts;
    st[19] = 0;   // engine: work list
    return 0;
}

// Verdicts of the shards a search ran on, and the record jtb_final_configs reads.  fc_valid = false: the visited
// table is not complete (scout-only test runs).
void set_verdicts(jtb_ctx* ctx, const jtb_history* h, const Prepared& P, const std::vector<int>& searchable, Search& r,
                  bool fc_valid, jtb_lin_shard* shards) {
    const int n_shards = h->n_shards;
    Ctrl& hc = r.hc;
    if (hc.stop == 2 && hc.cause == CAUSE_RING_FULL) hc.cause = JTB_CAUSE_BUDGET;
    if (hc.overflow) {   // a ring slot was overwritten before it was consumed: no verdict may be derived from this search
        hc.stop = 2;
        hc.cause = JTB_CAUSE_BUDGET;
        std::fill(r.found.begin(), r.found.end(), 0);
    }
    for (int s : searchable) {
        jtb_lin_shard& sh = shards[s];
        if (r.found[s]) {
            sh.valid = JTB_VALID;
        } else if (hc.stop == 2) {
            sh.valid = JTB_UNKNOWN;
            sh.cause = hc.cause;
        } else {
            sh.valid = JTB_INVALID;
            const int64_t g = r.max_rank[s];
            sh.witness_index = P.ret_index[g];
            if (g > P.rank_base[s]) sh.previous_ok_index = P.ret_index[g - 1];
        }
    }
    if (n_shards == 1) {
        shards[0].configs_explored = r.configs;
        shards[0].probes = r.probes;
    }
    ctx->fc.valid = fc_valid;
    ctx->fc.n_events = h->n_events;
    ctx->fc.n_shards = n_shards;
    ctx->fc.kw = P.key_words;
    ctx->fc.n_slots = r.n_slots;
    ctx->fc.max_rank = r.max_rank;
    ctx->fc.verdict.assign(n_shards, JTB_UNKNOWN);
    for (int s = 0; s < n_shards; ++s) ctx->fc.verdict[s] = shards[s].valid;
}

}  // namespace

extern "C" {

int jtb_abi_version(void) { return JTB_ABI_VERSION; }

long jtb_struct_size(int which) {
    switch (which) {
    case 0: return sizeof(jtb_history);
    case 1: return sizeof(jtb_model);
    case 2: return sizeof(jtb_opts);
    case 3: return sizeof(jtb_lin_shard);
    case 4: return sizeof(jtb_lin_result);
    case 5: return sizeof(jtb_setfull_shard);
    case 6: return sizeof(jtb_setfull_out);
    case 7: return sizeof(jtb_bank_result);
    case 8: return sizeof(jtb_final_config);
    case 9: return sizeof(jtb_mono_shard);
    case 10: return sizeof(jtb_mono_result);
    case 11: return sizeof(jtb_cb_shard);
    case 12: return sizeof(jtb_cb_result);
    case 13: return sizeof(jtb_tl_shard);
    case 14: return sizeof(jtb_tl_result);
    case 15: return sizeof(jtb_rx_shard);
    case 16: return sizeof(jtb_rx_result);
    case 17: return sizeof(jtb_rg_shard);
    case 18: return sizeof(jtb_rg_result);
    case 19: return sizeof(jtb_tp_shard);
    case 20: return sizeof(jtb_tp_result);
    case 21: return sizeof(jtb_sw_shard);
    case 22: return sizeof(jtb_sw_result);
    case 23: return sizeof(jtb_rw_shard);
    case 24: return sizeof(jtb_rw_result);
    case 25: return sizeof(jtb_lw_shard);
    case 26: return sizeof(jtb_lw_result);
    case 27: return sizeof(jtb_cw_shard);
    case 28: return sizeof(jtb_cw_result);
    case 30: return sizeof(jtb_lk_shard);
    case 31: return sizeof(jtb_lk_result);
    case 33: return sizeof(jtb_edn_history);
    case 34: return sizeof(jtb_edn_checks);
    }
    return -1;
}

int jtb_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) return -1;
    return n;
}

jtb_ctx* jtb_create(const jtb_opts* opts) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) return nullptr;
    jtb_ctx* ctx = new jtb_ctx();
    if (opts) ctx->opts = *opts;
    ctx->device = ctx->opts.device;
    if (ctx->device < 0 || ctx->device >= n || cudaSetDevice(ctx->device) != cudaSuccess) {
        delete ctx;
        return nullptr;
    }
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, ctx->device);
    ctx->n_sms = prop.multiProcessorCount;
    int prio_lo = 0, prio_hi = 0;
    cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithPriority(&ctx->scout_stream, cudaStreamNonBlocking, prio_hi) != cudaSuccess ||
        cudaEventCreate(&ctx->ev0) != cudaSuccess || cudaEventCreate(&ctx->ev1) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->ev_setup, cudaEventDisableTiming) != cudaSuccess) {
        delete ctx;
        return nullptr;
    }
    return ctx;
}

void jtb_destroy(jtb_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    DevBuf* bufs[] = {&ctx->table, &ctx->pool, &ctx->rows, &ctx->classes, &ctx->cls_inv, &ctx->ctrl, &ctx->found,
                      &ctx->maxrank, &ctx->sc_init, &ctx->sc_tables, &ctx->sc_stacks, &ctx->sc_ctl, &ctx->lv_ctrl,
                      &ctx->lv_buf[0], &ctx->lv_buf[1], &ctx->lv_aux[0], &ctx->lv_aux[1], &ctx->lv_beam};
    for (DevBuf* b : bufs)
        if (b->p) cudaFree(b->p);
    ctx->sf.release();
    if (ctx->ev0) cudaEventDestroy(ctx->ev0);
    if (ctx->ev1) cudaEventDestroy(ctx->ev1);
    if (ctx->ev_setup) cudaEventDestroy(ctx->ev_setup);
    if (ctx->scout_stream) cudaStreamDestroy(ctx->scout_stream);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    delete ctx;
}

const char* jtb_last_error(const jtb_ctx* ctx) { return ctx ? ctx->err.c_str() : "no context (no CUDA device?)"; }

// -------------------------------------------------------------------------------------------------
// force_worklist: search with the work-list engine whatever the options and the history say (its table then holds
// every visited configuration, which jtb_final_configs reads)
static int check_lin_impl(jtb_ctx* ctx, const jtb_history* h, const jtb_model* m, jtb_lin_shard* shards,
                          jtb_lin_result* out, bool force_worklist) {
    const double t_start = now_s();
    ctx->fc.valid = false;
    CK(cudaSetDevice(ctx->device));
    if (m->kind != JTB_MODEL_REGISTER && m->kind != JTB_MODEL_CAS_REGISTER && m->kind != JTB_MODEL_BANK &&
        m->kind != JTB_MODEL_SET) {
        ctx->err = "model not supported by the device search";
        return -2;
    }
    Prepared P;
    if (!prepare(h, m, P)) {
        ctx->err = "malformed history: " + P.error;
        return -3;
    }
    const int n_shards = h->n_shards;
    const int KW = P.key_words;
    const bool bank = m->kind == JTB_MODEL_BANK;
    const int EW = KW + (bank ? 4 : 0);
    std::memset(out, 0, sizeof *out);
    out->key_bytes = KW * 8;
    for (int s = 0; s < n_shards; ++s) {
        std::memset(&shards[s], 0, sizeof shards[s]);
        shards[s].witness_index = shards[s].previous_ok_index = -1;
        if (P.shard_cause[s]) {
            shards[s].valid = JTB_UNKNOWN;
            shards[s].cause = P.shard_cause[s];
        }
    }
    // initial configurations: one per shard that has completed ops
    std::vector<uint64_t> init_entries;
    std::vector<int> searchable;
    auto add_init = [&](int s) {
        searchable.push_back(s);
        std::vector<uint64_t> e(EW, 0);
        e[0] = KEY_VALID | ((uint64_t)(uint32_t)P.rank_base[s] << 32) |
               ((bank || m->kind == JTB_MODEL_SET) ? 0ull : (uint64_t)(uint32_t)m->init_value);
        if (bank)
            for (int i = 0; i < 4; ++i)
                e[KW + i] = (uint64_t)(uint32_t)m->init_balance[2 * i] |
                            ((uint64_t)(uint32_t)m->init_balance[2 * i + 1] << 32);
        init_entries.insert(init_entries.end(), e.begin(), e.end());
    };
    for (int s = 0; s < n_shards; ++s)
        if (!P.shard_cause[s] && P.rank_base[s + 1] != P.rank_base[s]) add_init(s);
    ctx->stats[10] = 0;
    ctx->stats[12] = ctx->stats[13] = ctx->stats[14] = 0;
    ctx->stats[15] = ctx->stats[16] = ctx->stats[17] = ctx->stats[18] = 0;
    Search r(n_shards);
    auto finish = [&](const Search& res) {
        for (int s = 0; s < n_shards; ++s) {
            out->valid = std::max(out->valid, shards[s].valid);
            out->n_failures += shards[s].valid != JTB_VALID;
        }
        out->configs_explored = res.configs;
        out->probes = res.probes;
        out->hbm_bytes_algorithmic = (uint64_t)KW * 8 * (res.probes + res.configs);
        out->seconds_kernel = res.kernel_s;
        out->seconds_total = now_s() - t_start;
        return 0;
    };
    if (searchable.empty()) return finish(r);
    if (upload(ctx, ctx->rows, P.rows) || upload(ctx, ctx->classes, P.classes) || upload(ctx, ctx->cls_inv, P.cls_inv_pos))
        return -1;
    if (ensure(ctx, ctx->ctrl, sizeof(Ctrl)) || ensure(ctx, ctx->found, n_shards * sizeof(int)) ||
        ensure(ctx, ctx->maxrank, n_shards * sizeof(int)))
        return -1;
    const bool eager_mode = !(ctx->opts.flags & JTB_OPT_NO_EAGER_READS);
    const bool scout_only = getenv("JTB_SCOUT_ONLY") != nullptr;   // test hook of the work-list engine
    // ---- beam first (single-key histories with crashed ops; measured on the 8-key C5 "monster": one beam shared by
    //      several keys starves most of them — 2 of 8 decided after 7.7e8 configurations — so many-key histories keep
    //      the work list + scouts): finds the linearization of a VALID history in a few
    //      thousand narrow levels where an exhaustive search visits 10^8..10^10 configurations; keys it decides are
    //      VALID, the others go on to the exhaustive engine below ------------------------------------------------
    std::vector<char> beam_found(n_shards, 0);
    double beam_kernel_s = 0;
    unsigned long long beam_configs = 0, beam_levels = 0, beam_attempts = 0, beam_decided = 0, beam_probes = 0;
    ctx->stats[20] = ctx->stats[21] = ctx->stats[22] = ctx->stats[23] = 0;
    if (P.max_nc > 0 && P.max_nc <= 64 * LV_CLS_WORDS && n_shards <= LV_BEAM_SHARDS && searchable.size() == 1 &&
        P.n_ranks < LV_MAX_RANKS && !force_worklist && !scout_only &&
        !(ctx->opts.flags & (JTB_OPT_NO_BEAM | JTB_OPT_ENGINE_LEVEL | JTB_OPT_ENGINE_WORKLIST))) {
        // A budgeted run of the work list first (16 M configurations, no scouts): easy histories — most
        // histories with a few crashed ops — end there, at the work list's latency; only what it leaves open gets
        // the beam ladder.
        const uint64_t probe_budget = 16ull << 20;
        Search probe(n_shards);
        if (int rc = search_worklist(ctx, h, m, P, searchable, init_entries,
                                     ctx->opts.max_configs ? std::min<uint64_t>(ctx->opts.max_configs, probe_budget) : probe_budget,
                                     /*scouts_on=*/false, t_start, probe))
            return rc;
        std::vector<jtb_lin_shard> ps(shards, shards + n_shards);
        set_verdicts(ctx, h, P, searchable, probe, true, ps.data());
        bool all = true;
        for (int s : searchable) all = all && ps[s].valid != JTB_UNKNOWN;
        if (all) {
            std::copy(ps.begin(), ps.end(), shards);
            return finish(probe);
        }
        uint32_t widths[3] = {256u, 2048u, 16384u};
        int n_widths = 3;
        if (const char* bw = getenv("JTB_BEAM_W")) { widths[0] = (uint32_t)std::max(1, atoi(bw)); n_widths = 1; }   // experiments
        for (int wi = 0; wi < n_widths && !searchable.empty(); ++wi) {
            Search b(n_shards);
            if (arm_shards(ctx, P, n_shards, b.max_rank)) return -1;
            if (int rc = search_level(ctx, m, P, n_shards, searchable, init_entries, b.hc, b.kernel_s, b.configs, b.probes, widths[wi]))
                return rc;
            CK(cudaMemcpyAsync(b.found.data(), ctx->found.p, n_shards * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
            CK(cudaStreamSynchronize(ctx->stream));
            beam_kernel_s += b.kernel_s; beam_configs += b.configs; beam_probes += b.probes; beam_levels += ctx->stats[2]; ++beam_attempts;
            std::vector<int> left;
            for (int s : searchable) {
                if (b.found[s]) { beam_found[s] = 1; ++beam_decided; }
                else left.push_back(s);
            }
            searchable.clear();
            init_entries.clear();
            for (int s : left) add_init(s);
        }
        ctx->stats[20] = beam_levels; ctx->stats[21] = beam_configs; ctx->stats[22] = beam_decided; ctx->stats[23] = beam_attempts;
        if (searchable.empty()) {   // every key decided by the beam
            r.kernel_s = beam_kernel_s; r.configs = beam_configs; r.probes = beam_probes;
            r.hc.stop = 1;
            ctx->stats[19] = 1;
            ctx->last_engine = 1;
        }
    }
    if (!searchable.empty()) {
        // ---- engine: level-synchronous sweep (jtb_level.cuh) or work list (jtb_wgl.cuh) ---------------------------
        // Default choice: histories with crashed ops -> work list (its depth-first
        // order + scouts find the linearization of a valid history long before a breadth-first sweep would);
        // Knossos-exact space -> level engine (higher throughput on wide levels, bounded memory);
        // eager reads (product default) -> the search is narrow unless ~every client always has an op in flight
        // (mean open ops per frontier row >= 26 of 32): narrow searches are a chain of short levels, where the work
        // list's dependent steps are cheaper than a grid barrier per level.
        bool use_level = P.max_nc == 0 && (!eager_mode || P.mean_open >= 26.0);
        if (ctx->opts.flags & JTB_OPT_ENGINE_LEVEL) use_level = true;
        if (ctx->opts.flags & JTB_OPT_ENGINE_WORKLIST) use_level = false;
        if (force_worklist || scout_only) use_level = false;
        if (P.n_ranks >= LV_MAX_RANKS || P.max_nc > 64) use_level = false;   // epoch tag bits / class mask width
        if (use_level) {
            if (arm_shards(ctx, P, n_shards, r.max_rank)) return -1;
            if (int rc = search_level(ctx, m, P, n_shards, searchable, init_entries, r.hc, r.kernel_s, r.configs, r.probes)) return rc;
            CK(cudaMemcpyAsync(r.found.data(), ctx->found.p, n_shards * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
            CK(cudaMemcpyAsync(r.max_rank.data(), ctx->maxrank.p, n_shards * sizeof(int), cudaMemcpyDeviceToHost, ctx->stream));
            CK(cudaStreamSynchronize(ctx->stream));
            ctx->last_configs = r.configs;
            ctx->last_engine = 1;
        } else if (int rc = search_worklist(ctx, h, m, P, searchable, init_entries, ctx->opts.max_configs,
                                            !(ctx->opts.flags & JTB_OPT_NO_SCOUTS), t_start, r)) {
            return rc;
        }
        r.kernel_s += beam_kernel_s;
    }
    for (int s = 0; s < n_shards; ++s)
        if (beam_found[s]) shards[s].valid = JTB_VALID;
    set_verdicts(ctx, h, P, searchable, r, !scout_only, shards);
    return finish(r);
}

int jtb_check_linearizable(jtb_ctx* ctx, const jtb_history* h, const jtb_model* m, jtb_lin_shard* shards,
                           jtb_lin_result* out) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    return check_lin_impl(ctx, h, m, shards, out, false);
}

// -------------------------------------------------------------------------------------------------
// knossos :configs for an INVALID shard: the visited configurations stuck at the witness (SURVEY §8(f) N4)
int jtb_final_configs(jtb_ctx* ctx, const jtb_history* h, const jtb_model* m, int32_t shard, jtb_final_config* out,
                      int32_t cap, int64_t* n_total) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    CK(cudaSetDevice(ctx->device));
    if (ctx->fc.valid && ctx->last_engine == 1 && h->n_events == ctx->fc.n_events && h->n_shards == ctx->fc.n_shards) {
        // the level engine keeps no visited set: search again with the work-list engine, whose table holds every
        // visited configuration (same verdict and witness; only asked for after an INVALID verdict)
        std::vector<jtb_lin_shard> tmp_shards((size_t)h->n_shards);
        jtb_lin_result tmp_out;
        if (int rc = check_lin_impl(ctx, h, m, tmp_shards.data(), &tmp_out, true)) return rc;
    }
    if (!ctx->fc.valid || h->n_events != ctx->fc.n_events || h->n_shards != ctx->fc.n_shards || shard < 0 ||
        shard >= h->n_shards) {
        ctx->err = "jtb_final_configs: call it directly after jtb_check_linearizable on the same history";
        return -2;
    }
    if (ctx->fc.verdict[shard] != JTB_INVALID) {
        ctx->err = "jtb_final_configs: the shard was not found INVALID";
        return -2;
    }
    Prepared P;
    if (!prepare(h, m, P) || P.key_words != ctx->fc.kw) {
        ctx->err = "jtb_final_configs: the history does not match the last search";
        return -3;
    }
    const int KW = P.key_words, RW = P.row_words, SW = slot_words(m->kind);
    const bool bank = m->kind == JTB_MODEL_BANK;
    const int64_t g = ctx->fc.max_rank[shard], base = P.rank_base[shard];
    // ---- gather the keys at rank g ------------------------------------------------------------------
    std::vector<uint64_t> keys;
    if (g == base) {   // the initial configuration is never inserted
        keys.assign(KW, 0);
        keys[0] = KEY_VALID | ((uint64_t)(uint32_t)base << 32) |
                  ((bank || m->kind == JTB_MODEL_SET) ? 0ull : (uint64_t)(uint32_t)m->init_value);
    }
    {
        DevBuf d_cnt, d_out;
        auto free_all = [&]() { if (d_cnt.p) cudaFree(d_cnt.p); if (d_out.p) cudaFree(d_out.p); d_cnt = DevBuf(); d_out = DevBuf(); };
        struct Guard { decltype(free_all)& f; ~Guard() { f(); } } guard{free_all};   // CK() returns early on errors
        if (ensure(ctx, d_cnt, 8)) return -1;
        const uint64_t* table = (const uint64_t*)ctx->table.p;
        unsigned long long total = 0;
        for (int pass = 0; pass < 2; ++pass) {
            const unsigned long long want = pass == 0 ? 0 : std::min<unsigned long long>(total, 1ull << 22);
            if (pass == 1 && want == 0) break;
            if (pass == 1 && ensure(ctx, d_out, want * KW * 8)) { free_all(); return -1; }
            CK(cudaMemsetAsync(d_cnt.p, 0, 8, ctx->stream));
            const int grid = ctx->n_sms * 8;
            if (int rc = dispatch_model_kw(ctx, m->kind, KW, [&](auto, auto K) {
                    table_collect_kernel<K()><<<grid, 256, 0, ctx->stream>>>(table, ctx->fc.n_slots, (uint32_t)g, (uint64_t*)d_out.p,
                                                                             want, (unsigned long long*)d_cnt.p);
                    return 0;
                }))
                return rc;
            CK(cudaGetLastError());
            CK(cudaMemcpyAsync(&total, d_cnt.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
            CK(cudaStreamSynchronize(ctx->stream));
            if (pass == 1) {
                const size_t off = keys.size();
                keys.resize(off + (size_t)want * KW);
                CK(cudaMemcpy(keys.data() + off, d_out.p, (size_t)want * KW * 8, cudaMemcpyDeviceToHost));
            }
        }
        free_all();
        *n_total = (int64_t)total + (g == base ? 1 : 0);
    }
    // ---- decode -----------------------------------------------------------------------------------------
    std::vector<int32_t> pos_index;   // client-event position inside the shard -> :index
    for (int64_t e = h->shard_off[shard]; e < h->shard_off[shard + 1]; ++e)
        if (h->process[e] >= 0) pos_index.push_back(h->index[e]);
    const int32_t* row = &P.rows[(size_t)g * RW];
    const int cls_base = row[11], ncls = row[12];
    int32_t prefix_bal[JTB_MAX_ACCOUNTS];
    for (int i = 0; i < JTB_MAX_ACCOUNTS; ++i) prefix_bal[i] = m->init_balance[i];
    auto apply = [](int32_t* bal, const int32_t* op, int times) {   // bank transfer record (x, y = amount, z, w)
        if ((op[0] & 0xff) != JTB_F_TRANSFER || (op[0] & OP_IMPOSSIBLE)) return;
        bal[op[2]] -= op[1] * times;
        bal[op[3]] += op[1] * times;
    };
    if (bank)
        for (int64_t gg = base; gg < g; ++gg) {   // every op that returned before the witness is linearized
            const int32_t* r = &P.rows[(size_t)gg * RW];
            apply(prefix_bal, r + ROW_EXTRA + r[13] * SW, 1);
        }
    std::vector<jtb_final_config> all(keys.size() / KW);
    for (size_t k = 0; k < all.size(); ++k) {
        const uint64_t* key = &keys[k * KW];
        jtb_final_config& c = all[k];
        std::memset(&c, 0, sizeof c);
        c.state = (bank || m->kind == JTB_MODEL_SET) ? 0 : (int32_t)(uint32_t)key[0];
        for (int i = 0; i < JTB_MAX_ACCOUNTS; ++i) c.balances[i] = bank ? prefix_bal[i] : 0;
        for (int t = 0; t < P.S_pad; ++t) {
            const int32_t* cell = row + ROW_EXTRA + t * SW;
            if (cell[0] < 0) continue;
            const bool is_read = (cell[0] & 0xff) == JTB_F_READ;
            const int32_t ipos = (bank && !is_read) ? cell[4] : cell[3];
            const int32_t idx = pos_index[ipos];
            if ((key[1] >> t) & 1ull) {
                c.linearized_open_index[c.n_linearized_open++] = idx;
                if (bank) apply(c.balances, cell, 1);
            } else {
                c.pending_index[c.n_pending++] = idx;
            }
        }
        std::sort(c.pending_index, c.pending_index + c.n_pending);
        std::sort(c.linearized_open_index, c.linearized_open_index + c.n_linearized_open);
        for (int cc = 0; cc < ncls; ++cc) {
            const ClassRec& cr = P.classes[cls_base + cc];
            const int shift = cr.shift_width & 0xff, width = cr.shift_width >> 8;
            const int count = (int)((key[cr.word] >> shift) & ((1ull << width) - 1));
            c.n_crashed_linearized += count;
            if (bank) apply(c.balances, &cr.op.x, count);
        }
    }
    // canonical order: lexicographic over the struct's int32 fields in declaration order (unused entries are 0)
    std::sort(all.begin(), all.end(), [](const jtb_final_config& a, const jtb_final_config& b) {
        const int32_t* x = reinterpret_cast<const int32_t*>(&a);
        const int32_t* y = reinterpret_cast<const int32_t*>(&b);
        for (size_t i = 0; i < sizeof(jtb_final_config) / 4; ++i)
            if (x[i] != y[i]) return x[i] < y[i];
        return false;
    });
    const size_t n_out = std::min<size_t>(all.size(), (size_t)std::max(cap, 0));
    if (n_out) std::memcpy(out, all.data(), n_out * sizeof(jtb_final_config));
    return 0;
}

// -------------------------------------------------------------------------------------------------
int jtb_check_set_full(jtb_ctx* ctx, const jtb_history* h, int linearizable, jtb_setfull_out* out) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    return run_set_full(ctx->stream, ctx->ev0, ctx->ev1, ctx->sf, h, linearizable, out, ctx->err, ctx->stats);
}

int jtb_check_bank_totals(jtb_ctx* ctx, const jtb_history* h, const jtb_model* accounts, int64_t total_amount,
                          jtb_bank_result* out) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    return run_bank_totals(ctx->stream, ctx->ev0, ctx->ev1, h, accounts, total_amount, out, ctx->err);
}

// K7: the monotonic-key check (csrc/jtb_monotonic.cuh)
int jtb_check_monotonic_keys(jtb_ctx* ctx, const jtb_history* h, int32_t flags, jtb_mono_shard* shards,
                             jtb_mono_result* out) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    return run_monotonic_keys(ctx->stream, ctx->ev0, ctx->ev1, h, flags, shards, out, ctx->err);
}

// K8: the counter-bounds check (csrc/jtb_counter_bounds.cuh)
int jtb_check_counter_bounds(jtb_ctx* ctx, const jtb_history* h, int32_t flags, jtb_cb_shard* shards,
                             jtb_cb_result* out) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    return run_counter_bounds(ctx->stream, ctx->ev0, ctx->ev1, h, flags, shards, out, ctx->err);
}

// K9: the transfer-lookup check (csrc/jtb_transfer_lookups.cuh)
int jtb_check_transfer_lookups(jtb_ctx* ctx, const jtb_history* h, int32_t flags, jtb_tl_shard* shards,
                               jtb_tl_result* out) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    return run_transfer_lookups(ctx->stream, ctx->ev0, ctx->ev1, h, flags, shards, out, ctx->err);
}

// K10: the read-explanation check (csrc/jtb_read_explanations.cuh)
int jtb_check_read_explanations(jtb_ctx* ctx, const jtb_history* h, int64_t max_nodes, int32_t flags,
                                jtb_rx_shard* shards, jtb_rx_result* out) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    return run_read_explanations(ctx->stream, ctx->ev0, ctx->ev1, h, max_nodes, flags, shards, out, ctx->err);
}

// K11: the read-gap check (csrc/jtb_read_gaps.cuh)
int jtb_check_read_gaps(jtb_ctx* ctx, const jtb_history* h, int64_t max_nodes, int32_t flags, jtb_rg_shard* shards,
                        jtb_rg_result* out) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    return run_read_gaps(ctx->stream, ctx->ev0, ctx->ev1, h, max_nodes, flags, shards, out, ctx->err);
}

// K12: the transfer-placement check (csrc/jtb_transfer_placement.cuh)
int jtb_check_transfer_placement(jtb_ctx* ctx, const jtb_history* h, int64_t max_nodes, int32_t max_rounds,
                                 int32_t flags, jtb_tp_shard* shards, jtb_tp_result* out) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    return run_transfer_placement(ctx->stream, ctx->ev0, ctx->ev1, h, max_nodes, max_rounds, flags, shards, out,
                                  ctx->err);
}

// K13: the serial-witness check (csrc/jtb_serial_witness.cuh)
int jtb_check_serial_witness(jtb_ctx* ctx, const jtb_history* h, int64_t max_nodes, int32_t max_rounds, int32_t flags,
                             int32_t* commit_read, jtb_sw_shard* shards, jtb_sw_result* out) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    return run_witness_as(ctx->stream, ctx->ev0, ctx->ev1, h, max_nodes, max_rounds, 0, 0, flags, commit_read, shards,
                          out, ctx->err);
}

// K14: the repaired serial witness (csrc/jtb_repaired_witness.cuh)
int jtb_check_repaired_witness(jtb_ctx* ctx, const jtb_history* h, int64_t max_nodes, int32_t max_rounds,
                               int32_t max_repairs, int32_t flags, int32_t* commit_read, jtb_rw_shard* shards,
                               jtb_rw_result* out) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    if (max_repairs <= 0) max_repairs = JTB_RW_DEFAULT_MAX_REPAIRS;
    return run_witness_as(ctx->stream, ctx->ev0, ctx->ev1, h, max_nodes, max_rounds, max_repairs, 0, flags,
                          commit_read, shards, out, ctx->err);
}

// K15: the lifted serial witness (csrc/jtb_lifted_witness.cuh)
int jtb_check_lifted_witness(jtb_ctx* ctx, const jtb_history* h, int64_t max_nodes, int32_t max_rounds,
                             int32_t max_repairs, int32_t max_lifts, int32_t flags, int32_t* commit_read,
                             jtb_lw_shard* shards, jtb_lw_result* out) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    if (max_repairs <= 0) max_repairs = JTB_RW_DEFAULT_MAX_REPAIRS;
    if (max_lifts <= 0) max_lifts = JTB_LW_DEFAULT_MAX_LIFTS;
    return run_witness_as(ctx->stream, ctx->ev0, ctx->ev1, h, max_nodes, max_rounds, max_repairs, max_lifts, flags,
                          commit_read, shards, out, ctx->err);
}

// K16: the class witness (csrc/jtb_class_witness.cuh)
int jtb_check_class_witness(jtb_ctx* ctx, const jtb_history* h, int64_t max_nodes, int32_t max_rounds,
                            int32_t max_repairs, int32_t max_lifts, int32_t flags, int32_t* commit_read,
                            jtb_cw_shard* shards, jtb_cw_result* out) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    if (max_repairs <= 0) max_repairs = JTB_RW_DEFAULT_MAX_REPAIRS;
    if (max_lifts <= 0) max_lifts = JTB_LW_DEFAULT_MAX_LIFTS;
    return run_witness_as(ctx->stream, ctx->ev0, ctx->ev1, h, max_nodes, max_rounds, max_repairs, max_lifts, flags,
                          commit_read, shards, out, ctx->err, CwPass{});
}

// K17: the lookup witness (csrc/jtb_lookup_witness.cuh)
int jtb_check_lookup_witness(jtb_ctx* ctx, const jtb_history* h, int64_t max_nodes, int32_t max_rounds,
                             int32_t max_repairs, int32_t max_lifts, int32_t flags, int32_t* commit_read,
                             int32_t* lookup_read, jtb_lk_shard* shards, jtb_lk_result* out) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    if (max_repairs <= 0) max_repairs = JTB_RW_DEFAULT_MAX_REPAIRS;
    if (max_lifts <= 0) max_lifts = JTB_LW_DEFAULT_MAX_LIFTS;
    LkPass pass;
    pass.lookup_read = lookup_read;
    return run_witness_as(ctx->stream, ctx->ev0, ctx->ev1, h, max_nodes, max_rounds, max_repairs, max_lifts, flags,
                          commit_read, shards, out, ctx->err, pass);
}

// K18: a stored ledger history.edn read on the device (csrc/jtb_edn.cuh)
int jtb_read_ledger_edn(jtb_ctx* ctx, const char* text, int64_t n_bytes, int32_t form, int32_t flags,
                        jtb_edn_history* out) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    return run_read_ledger_edn(ctx->stream, ctx->ev0, ctx->ev1, text, n_bytes, form, flags, out, ctx->err);
}

void jtb_edn_history_free(jtb_edn_history* out) {
    if (out) jtb_edn_history_release(out);
}

// K19: the host checks of a ledger compose on a stored history.edn (csrc/jtb_edn_checks.cuh)
int jtb_ledger_edn_checks(jtb_ctx* ctx, const char* text, int64_t n_bytes, int32_t flags, jtb_edn_checks* out) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    return run_ledger_edn_checks(ctx->stream, ctx->ev0, ctx->ev1, text, n_bytes, flags, out, ctx->err);
}

void jtb_edn_checks_free(jtb_edn_checks* out) {
    if (out) jtb_edn_checks_release(out);
}

// K20: a stored set-full history.edn read on the device (csrc/jtb_set_edn.cuh)
int jtb_read_set_edn(jtb_ctx* ctx, const char* text, int64_t n_bytes, int32_t flags, jtb_edn_history* out) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    return run_read_set_edn(ctx->stream, ctx->ev0, ctx->ev1, text, n_bytes, flags, out, ctx->err);
}

// SURVEY 8(f) N2: the step before the checkers (independent/subhistory, ledger->bank) on the device
int jtb_partition_by_key(jtb_ctx* ctx, int64_t n_events, const int64_t* event_key, int32_t* order, int64_t* shard_off,
                         int64_t* key_ids, int32_t key_cap, int32_t* n_keys) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    return run_partition_by_key(ctx->stream, n_events, event_key, order, shard_off, key_ids, key_cap, n_keys, ctx->err);
}

int jtb_ledger_balances(jtb_ctx* ctx, int64_t n, const int64_t* credits_posted, const int64_t* debits_posted, int32_t* balance) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    return run_ledger_balances(ctx->stream, n, credits_posted, debits_posted, balance, ctx->err);
}

// Page-locked host memory for the caller's flattened arrays (the id lists of set-full reads are hundreds of MB: from
// pageable memory the H2D copy is staged through the driver's bounce buffers at a fraction of the PCIe rate).
void* jtb_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 16, cudaHostAllocDefault) != cudaSuccess) { (void)cudaGetLastError(); return nullptr; }
    return p;
}

void jtb_host_free(void* p) {
    if (p) cudaFreeHost(p);
}

double jtb_prepare_seconds(const jtb_history* h, const jtb_model* m) {
    const double t0 = now_s();
    Prepared P;
    if (!prepare(h, m, P)) return -1.0;
    return now_s() - t0;
}

double jtb_prepare_info(const jtb_history* h, const jtb_model* m, long long info[4]) {
    const double t0 = now_s();
    Prepared P;
    if (!prepare(h, m, P)) return -1.0;
    info[0] = P.key_words * 8; info[1] = P.S_pad; info[2] = P.max_nc; info[3] = P.n_ranks;
    return now_s() - t0;
}

int jtb_get_stats(jtb_ctx* ctx, unsigned long long* out, int n) {
    if (!ctx) return -1;
    for (int i = 0; i < n && i < 24; ++i) out[i] = ctx->stats[i];
    return 0;
}

int jtb_table_bench(jtb_ctx* ctx, uint64_t n_keys, int variant, int rounds, double* insert_seconds,
                    double* probe_seconds, uint64_t* found) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    size_t table_bytes = ctx->opts.table_bytes ? ctx->opts.table_bytes : (size_t)8 << 30;
    uint64_t n_slots = 1;
    while (n_slots * 2 * 16 <= table_bytes) n_slots <<= 1;
    if (ensure(ctx, ctx->table, n_slots * 16)) return -1;
    return run_table_bench(ctx->stream, ctx->ev0, ctx->ev1, (uint64_t*)ctx->table.p, n_slots, n_keys, variant, rounds,
                           ctx->n_sms, insert_seconds, probe_seconds, found, ctx->err);
}

int jtb_gather_bench(jtb_ctx* ctx, uint64_t table_bytes, int in_flight, int wide, uint32_t iters, int ctas_per_sm,
                     int rounds, double* seconds, uint64_t* n_probes) {
    if (!ctx) return -1;
    std::lock_guard<std::mutex> lk(ctx->mu);
    if (cudaSetDevice(ctx->device) != cudaSuccess) { ctx->err = "cudaSetDevice failed"; return -1; }
    ctx->fc.valid = false;
    uint64_t n_slots = 1;
    while (n_slots * 2 * 16 <= table_bytes) n_slots <<= 1;
    if (ensure(ctx, ctx->table, n_slots * 16)) return -1;
    return run_gather_bench(ctx->stream, ctx->ev0, ctx->ev1, (uint64_t*)ctx->table.p, n_slots, in_flight, wide, iters,
                            std::max(1, ctas_per_sm), std::max(1, rounds), ctx->n_sms, seconds, n_probes, ctx->err);
}

}  // extern "C"
