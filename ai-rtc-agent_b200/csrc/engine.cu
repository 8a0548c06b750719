// Per-frame engine: VAE encoder (TAESD, or the model's AutoencoderKL) -> stream-batched UNet -> LCM step -> VAE decoder, assembled once
// (at b2sd_prepare) as a static list of kernel launches over preallocated HBM buffers and replayed as
// a CUDA graph.  Mirrors what the reference reaches through StreamDiffusion.__call__
// (lib/wrapper.py:330) and its three TensorRT engines (lib/wrapper.py:445-466).
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <functional>
#include <thread>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/b200sd.h"
#include "attention.cuh"
#include "canny.cuh"
#include "elementwise.cuh"
#include "igemm.cuh"
#include "tconv.cuh"

using namespace b2;

namespace b2 {
// capi.cu: a contraction as launched, in the C ABI's terms (plan = NULL: the halo-tile kernel)
void igemm_record(const IgemmDesc& g, const IgemmPlan* plan, b2sd_igemm_desc* d, b2sd_igemm_plan_info* info);
}

#define CUDA_OK(expr)                                                                       \
    do {                                                                                    \
        cudaError_t e__ = (expr);                                                           \
        if (e__ != cudaSuccess) {                                                           \
            b2_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
            return -1;                                                                      \
        }                                                                                   \
    } while (0)
#define TRY(expr)            \
    do {                     \
        if ((expr) != 0) return -1; \
    } while (0)

namespace {

struct Act {
    __half* p = nullptr;
    int n = 0, h = 0, w = 0, c = 0, ld = 0;
    long elems() const { return (long)n * h * w * ld; }
};

struct Raw {  // a loaded parameter, fp16 on device (+ host fp32 copy for 1-D tensors)
    __half* p = nullptr;      // null once released (pack-only parameters after the first successful prepare)
    bool pack_only = false;   // only ever read by the packing kernels (3x3 / shortcut convs, q/k/v, GEGLU, Cin<=4 convs)
    bool derived = false;     // computed by the engine from loaded parameters (exact weight foldings): dropped on any reload
    std::vector<int64_t> shape;
    std::vector<float> host;
    long numel() const {
        long v = 1;
        for (auto s : shape) v *= s;
        return v;
    }
};

// bump allocator over cudaMalloc'ed slabs (HBM is plentiful: no reuse, no fragmentation)
class Arena {
  public:
    explicit Arena(size_t slab) : slab_(slab) {}
    ~Arena() { release(); }
    // Stream-ordered mode (a style's store and lanes, b2sd_create_style): slabs come from `pool` on `order` and are freed on
    // it, so releasing them never synchronises the device; whoever frees first makes `order` wait for the last work that
    // reads them (b2sd_release).  The pool must not reuse memory across streams by waiting (no internal dependencies): the
    // host waits for each allocation, and so would wait for the frames of whatever stream freed it.  Set before the first alloc.
    void set_order(cudaStream_t order, cudaMemPool_t pool) { order_ = order; pool_ = pool; }
    void* alloc(size_t bytes) {
        bytes = (bytes + 1023) & ~size_t(1023);
        if (cur_ < 0 || off_ + bytes > sizes_[cur_]) {
            // find next slab that fits, else allocate
            int next = cur_ + 1;
            while (next < (int)slabs_.size() && sizes_[next] < bytes) ++next;
            if (next >= (int)slabs_.size()) {
                size_t sz = bytes > slab_ ? bytes : slab_;
                void* p = nullptr;
                cudaError_t e = order_ ? cudaMallocFromPoolAsync(&p, sz, pool_, order_) : cudaMalloc(&p, sz);
                if (e == cudaSuccess && order_) e = cudaStreamSynchronize(order_);   // usable on any stream from here on
                if (e != cudaSuccess) {   // callers only see nullptr: say why, or the caller reports a stale message
                    b2_set_error("device allocation of %zu bytes failed: %s", sz, cudaGetErrorString(e));
                    return nullptr;
                }
                slabs_.push_back(p);
                sizes_.push_back(sz);
                next = (int)slabs_.size() - 1;
            }
            cur_ = next;
            off_ = 0;
        }
        void* r = static_cast<char*>(slabs_[cur_]) + off_;
        off_ += bytes;
        return r;
    }
    void reset() { cur_ = slabs_.empty() ? -1 : 0; off_ = 0; }
    void release() {
        for (void* p : slabs_) order_ ? cudaFreeAsync(p, order_) : cudaFree(p);
        slabs_.clear();
        sizes_.clear();
        cur_ = -1;
        off_ = 0;
    }

  private:
    size_t slab_;
    cudaStream_t order_ = nullptr;
    cudaMemPool_t pool_ = nullptr;
    std::vector<void*> slabs_;
    std::vector<size_t> sizes_;
    int cur_ = -1;
    size_t off_ = 0;
};

struct Op {
    std::function<int(cudaStream_t)> fn;
    std::string name;
    double flops = 0.0;  // algorithmic 2*MAC count of the launch (0 for non-contraction kernels)
    b2sd_launch_record rec{};   // what the launch computes (b2sd_audit_step / _refresh); set where it is pushed
    template <class F>
    Op(F f, std::string n = "", double fl = 0.0) : fn(std::move(f)), name(std::move(n)), flops(fl) {}
    template <class F>
    Op(F f, std::string n, const b2sd_launch_record& r) : fn(std::move(f)), name(std::move(n)), rec(r) {}
    int operator()(cudaStream_t s) const { return fn(s); }
};

// Launch records of the elementwise kernels: the launcher's arguments in the C ABI's terms
b2sd_launch_record smallconv_record(const SmallConvArgs& a) {
    b2sd_launch_record r{};
    r.kind = B2SD_LAUNCH_SMALLCONV;
    r.smallconv = b2sd_smallconv_args{a.x, a.wt, a.bias, a.y, a.ldy, a.nb, a.h, a.w_, a.cin, a.cout, a.in_h, a.in_w, a.flags,
                                      a.res, a.ldr, (int64_t)a.res_bstride, a.in_off};
    return r;
}
b2sd_launch_record upsample2x_record(const void* x, void* y, int nb, int h, int w, int c) {
    b2sd_launch_record r{};
    r.kind = B2SD_LAUNCH_UPSAMPLE2X;
    r.upsample2x = b2sd_upsample2x_args{x, y, nb, h, w, c};
    return r;
}
b2sd_launch_record post_u8_record(const void* y, int ldy, void* out, int nb, int h, int w) {
    b2sd_launch_record r{};
    r.kind = B2SD_LAUNCH_POST_U8;
    r.post_u8 = b2sd_post_u8_args{y, ldy, out, nb, h, w};
    return r;
}
b2sd_launch_record small_linear_record(const float* in, int in_ld, const void* w, const float* bias, float* out, int out_ld,
                                       int nb, int n, int k, int silu_in) {
    b2sd_launch_record r{};
    r.kind = B2SD_LAUNCH_SMALL_LINEAR;
    r.small_linear = b2sd_small_linear_args{in, in_ld, w, bias, out, out_ld, nb, n, k, silu_in};
    return r;
}

}  // namespace

// ------------------------------------------------------------------------------------------------
// Tile / split-K policy of the frame program (batch-1 driven; derived from a cold-weight sweep of the contractions with
// tools/bench_op.py, not from a model).  Fills `plan` for the chosen (BN, splits, orientation).
// allow_swap: the caller is a UNet contraction (never TAESD / V^T / GEGLU).  Host-only: works in igemm dry-run mode.
static int igemm_autotile_single(IgemmDesc d, bool allow_swap, IgemmPlan* plan_out);

// Tile policy + CTA pairs.  The single-CTA policy picks orientation, N tile and split-K.  With d.pair_auto (set by the engine
// when several frames are in flight) a normal-orientation result with >= 2 M tiles and an N tile that is a multiple of 32 is
// re-planned as CTA pairs (2-CTA clusters) with the same N tile and the split-K factor capped at d.pair_splits: under
// concurrency the GPU is filled by the other frames, so what counts is SM time per contraction, and a pair fetches half the
// weight bytes per SM from L2 (multicast) and needs no cluster reduction.  Tuning overrides: B2_PAIR=0/1/2, B2_PAIR_SPLITS=n, B2_PAIR_SINGLE=1 (control: re-plan
// with the capped split-K but single CTAs).
int igemm_autotile(IgemmDesc d, bool allow_swap, IgemmPlan* plan_out) {
    TRY(igemm_autotile_single(d, allow_swap, plan_out));
    static const char* pair_env = getenv("B2_PAIR");
    static const char* ps_env = getenv("B2_PAIR_SPLITS");
    static const bool pair_single = getenv("B2_PAIR_SINGLE") != nullptr;
    const int pair_mode = pair_env ? atoi(pair_env) : d.pair_auto;
    const int pair_splits = ps_env ? atoi(ps_env) : (d.pair_splits > 0 ? d.pair_splits : 4);
    const IgemmPlan& pl = *plan_out;
    const int m_tiles = pl.p.tiles_w * pl.p.tiles_h * pl.p.tiles_n;
    if (pair_mode <= 0 || pl.p.swap || m_tiles < 2 || (pl.p.BN % 32) != 0 || (d.epi.flags & (IG_SILU | IG_PAD0))) return 0;
    if (pair_mode == 2 && pl.p.total_kb < 20) return 0;
    d.swap = 0; d.BN = pl.p.BN; d.splits = pl.splits > pair_splits ? pair_splits : pl.splits; d.partial = nullptr;
    d.pair = pair_single ? 0 : 1;
    IgemmPlan paired;
    if (igemm_plan(d, &paired)) return 0;   // keep the single-CTA plan
    *plan_out = paired;
    return 0;
}

static int igemm_autotile_single(IgemmDesc d, bool allow_swap, IgemmPlan* plan_out) {
    IgemmPlan& plan = *plan_out;
    const bool geglu = (d.epi.flags & IG_GEGLU) != 0;
    const bool silu = (d.epi.flags & IG_SILU) != 0;   // SiLU-epilogue kernels exist for N tiles of 16..128 only
    const bool pad0 = (d.epi.flags & IG_PAD0) != 0;   // tap-origin-0 kernels: N tiles of 64 / 128 / 256, normal orientation
    const int n_gemm = geglu ? 2 * d.epi.n_valid : d.epi.n_valid;
    static const bool swap_on = getenv("B2_SWAP") != nullptr, swap_off = getenv("B2_NO_SWAP") != nullptr;
    static const bool tuned = getenv("B2_NO_TUNED_TILES") == nullptr;
    static const char* ms_env = getenv("B2_MAX_SPLITS");   // tuning: cap of the cluster split-K factor (throughput vs latency)
    const int max_splits = ms_env ? atoi(ms_env) : (d.max_splits > 0 ? d.max_splits : 8);
    int total_kb = 0;
    for (int sidx = 0; sidx < d.nseg && sidx < IG_MAX_SRC; ++sidx) total_kb += d.ntap[sidx] * (d.src[sidx].C / IG_BK);
    const long rows_all = (long)d.Nb * d.Ho * d.Wo;
    // Swapped orientation by default only where it measured faster (tools/bench_op.py, cold weights): the 8x8 level,
    // where a 128-pixel M tile would be half empty.  B2_SWAP=1 forces it for every eligible UNet contraction.
    const bool swap_here = allow_swap && !geglu && !pad0 && !d.epi.acc_scale_b && d.epi.n_valid >= 128 && (d.epi.n_valid & 7) == 0 &&
                           (swap_on || (!swap_off && tuned && rows_all <= 64 && total_kb >= 90));
    if (swap_here) {
        d.swap = 1;
        d.BN = rows_all >= 256 ? 256 : (rows_all >= 128 ? 128 : 64);
        d.splits = 1; d.partial = nullptr;
        TRY(igemm_plan(d, &plan));
        const long ctas = (long)plan.grid.x * plan.grid.y;
        int max_by_k = plan.p.total_kb / 4;
        if (max_by_k < 1) max_by_k = 1;
        if (max_by_k > 8) max_by_k = 8;
        int splits = 1;
        while (splits * 2 <= max_by_k && ctas * splits * 2 <= 192 && splits * 2 <= max_splits) splits *= 2;
        if (splits > 1) {
            d.splits = splits;
            TRY(igemm_plan(d, &plan));
        }
        return 0;
    }
    d.swap = 0;
    auto vt_ok = [&](int bn) { return !d.epi.out2 || d.epi.col2 % bn == 0; };   // fused q/k/v: an N tile is all q/k or all v
    if (tuned && !geglu && !silu && !pad0 && n_gemm % 160 == 0 && total_kb >= 40 && vt_ok(160)) {
        // K-heavy contractions that cannot fill the GPU with 160-wide tiles alone (batch 1): wide tiles + cluster
        // split-K beat 64-wide tiles (weights streamed from HBM)
        d.BN = 160; d.splits = 1; d.partial = nullptr;
        TRY(igemm_plan(d, &plan));
        const int m_tiles = plan.p.tiles_w * plan.p.tiles_h * plan.p.tiles_n;
        const long tiles = (long)m_tiles * (n_gemm / 160);
        int bn = 0, splits = 0;
        if (tiles < 132) {
            if (m_tiles >= 8) { bn = 160; splits = 4; }
            else if (m_tiles >= 2 && n_gemm % 256 == 0 && total_kb >= 180 && vt_ok(256)) { bn = 256; splits = 8; }
        }
        if (bn && splits > max_splits) bn = 0;   // capped: fall through to the generic choice below
        if (bn) {
            d.BN = bn; d.splits = splits;
            TRY(igemm_plan(d, &plan));
            return 0;
        }
    }
    static const int cands[] = {256, 160, 128, 64, 32, 16};
    std::vector<int> valid;
    for (int bn : cands) {
        if (geglu && (bn % 32 != 0 || bn < 64)) continue;
        if (silu && (bn > 128 || bn % 16 || (bn & (bn - 1)))) continue;
        if (pad0 && bn != 64 && bn != 128 && bn != 256) continue;
        if (n_gemm % bn == 0 && vt_ok(bn)) valid.push_back(bn);
    }
    if (valid.empty()) {  // ragged N: one masked tile size
        int bn = 16;
        while (bn < n_gemm && bn < 128) bn <<= 1;
        valid.push_back(bn);
    }
    for (int bn : valid) {
        if (bn < 64 && n_gemm >= 64) break;  // narrow tiles re-read A too often: prefer split-K below
        d.BN = bn; d.splits = 1; d.partial = nullptr;
        TRY(igemm_plan(d, &plan));
        if (plan.p.acc_bufs == 2 || (long)plan.grid.x * plan.grid.y >= b2_device_sms()) return 0;   // persistent = a full wave
    }
    // not enough tiles for one wave: smallest reasonable tile, then split K
    int bn = valid.back();
    for (int v : valid) if (v >= 64) bn = v;  // smallest >= 64 if any (valid is descending)
    d.BN = bn; d.splits = 1; d.partial = nullptr;
    TRY(igemm_plan(d, &plan));
    const long ctas = (long)plan.grid.x * plan.grid.y;
    int splits = ctas >= 96 ? 1 : (int)((IG_SMS + ctas - 1) / ctas);
    if (tuned && ctas >= 64 && total_kb <= 12) splits = 1;   // the cluster reduction (~3 us) costs more than 5 k-blocks
    const int max_by_k = plan.p.total_kb / 4 > 0 ? plan.p.total_kb / 4 : 1;
    if (splits > max_by_k) splits = max_by_k;
    if (splits > 8) splits = 8;
    while (splits > max_splits && splits > 1) splits >>= 1;
    if (geglu) splits = 1;
    if (splits > 1) {
        d.splits = splits;
        TRY(igemm_plan(d, &plan));
    }
    return 0;
}

// Parameters and everything derived from them (kernel-native packed layouts, fused fp32 vectors).  Read-only on the frame
// path, so several engines ("lanes", b2sd_create_lane) share one store: one copy of the 1.7 GB UNet in HBM however many
// frames are in flight.
struct WeightStore {
    // ---- styles (b2sd_create_style).  Declared first, so destroyed last: the arenas below free on `order`, and a style reads
    // its parent's base values until then.
    std::shared_ptr<WeightStore> parent;   // a style: the live store whose base values it reads in place
    struct OrderStream {
        cudaStream_t s = nullptr;
        cudaMemPool_t pool = nullptr;
        ~OrderStream() {
            if (s) cudaStreamDestroy(s);         // returns at once; the frees queued on it still run
            if (pool) cudaMemPoolDestroy(pool);  // released once its last allocation is freed
        }
    } order;                               // a style: the stream and pool its memory is allocated and freed with
    const uint64_t id = next_id();         // tells the stores apart (the overrides computed with their parameters)
    uint64_t family = id;                  // a store and the styles derived from it: their states may move between them
    struct Copy { __half* dst; const __half* src; size_t bytes; };
    std::vector<Copy> pending;             // a style: base values copied into its own matrices by its first prepare
    static uint64_t next_id() {
        static std::atomic<uint64_t> n{1};
        return n++;
    }

    std::map<std::string, Raw> raw;
    Arena weights{256u << 20};   // packed parameters + the raw ones kernels read directly (live for the store's lifetime)
    Arena raw_only{256u << 20};  // raw parameters that only feed the packing kernels: released after the first prepare
    bool raw_released = false;
    bool imported = false;       // parameters came from a packed blob (b2sd_import_packed)
    std::map<std::string, __half*> packed;   // cache of packed weight matrices
    std::map<std::string, float*> fvec;      // cache of fp32 vectors
    std::map<std::string, size_t> packed_bytes, fvec_bytes;   // their sizes (b2sd_export_packed)
    std::shared_ptr<struct CondPool> cond_pool;   // made by the first conditioning override of a state of this store

    // ---- live parameters (b2sd_set_live_params / b2sd_apply_lora) ----
    // How each packed / fp32-vector cache entry derived from raw parameters is rebuilt in place: recorded when it is first
    // made (in every mode; it is host state only).  `keys` are the raw parameters it reads through src().
    struct Rebuild {
        std::vector<std::string> keys;
        std::function<int(cudaStream_t)> fn;
    };
    std::map<std::string, Rebuild> rebuild;
    std::map<std::string, const __half*> src_override;   // during b2sd_apply_lora: fused matrices the rebuilds read instead
    const __half* src(const std::string& key) const {
        auto o = src_override.find(key);
        if (o != src_override.end()) return o->second;
        auto it = raw.find(key);
        return it == raw.end() ? nullptr : it->second.p;
    }
    bool live = false;           // keep the base parameters; parameters may be re-fused at run time
    bool live_ready = false;     // the first prepare has made the base copies below
    Arena base_arena{256u << 20};
    std::map<std::string, __half*> base;   // base values of the UNet matrices kernels read raw (their live copy is raw[key].p)
    std::vector<std::string> fused;        // keys whose live values differ from the base (the last b2sd_apply_lora)
    void* scratch = nullptr;               // factor operands and fused matrices of b2sd_apply_lora, grown stream-ordered
    size_t scratch_cap = 0;
    ~WeightStore() {
        if (scratch) order.s ? cudaFreeAsync(scratch, order.s) : cudaFree(scratch);
    }
};

enum { COND_PROMPT = 0, COND_TIME = 1 };
static const uint64_t COND_GLOBAL = 0, COND_UNKNOWN = ~0ull;   // what a lane's block holds, besides an override's id

// Where the conditioning overrides of a weight store's states live and are freed.  The pool never makes an allocation wait for
// a free on another stream (no internal dependencies), and the frees run on a stream of their own: so neither the update that
// replaces an override nor the next one ever makes a lane's stream wait for the frames queued on another lane.
struct CondPool {
    cudaMemPool_t pool = nullptr;
    cudaStream_t reaper = nullptr;
    ~CondPool() {
        if (reaper) cudaStreamDestroy(reaper);   // returns at once; pending frees still run
        if (pool) cudaMemPoolDestroy(pool);      // released once its last allocation is freed
    }
};

// One state's own copy of one conditioning block (b2sd_state_set_prompt_embeds / _set_timesteps).  Immutable once published: an
// update makes a new one, since a lane that is behind on the device may still copy out of the old one.  The destructor frees it
// on the pool's reaper stream after the copy that computed it and after the latest copy out of it on every stream.
struct CondOverride {
    uint64_t id = 0;
    uint64_t store = 0;            // WeightStore::id of the parameters it was computed with
    bool own_text = false;         // a prompt block from the state's own prompt embeddings (else from the global ones)
    bool own_time = false;         // a time block whose time biases are from the state's own timesteps (else the global ones)
    bool own_control = false;      // ... and whose ControlNet scales are the state's own (else the global ones)
    void* buf = nullptr;
    size_t bytes = 0;
    cudaEvent_t ready = nullptr;   // recorded once buf holds the block
    std::vector<std::pair<cudaStream_t, cudaEvent_t>> uses;   // per stream, recorded after its latest copy out of buf
    std::shared_ptr<CondPool> pool;
    ~CondOverride() {
        if (!pool) return;   // the pool could not be made: nothing was allocated
        const cudaStream_t r = pool->reaper;
        if (ready) cudaStreamWaitEvent(r, ready, 0);
        for (auto& u : uses) {
            cudaStreamWaitEvent(r, u.second, 0);
            cudaEventDestroy(u.second);
        }
        if (buf) cudaFreeAsync(buf, r);
        if (ready) cudaEventDestroy(ready);
    }
};

// One temporal stream's stream-batch state (b2sd_state_*): slots 1 .. T-1 of the UNet input batch, NHWC fp16, stream-ordered
// allocation.  It remembers the family of weight stores (a store and its styles), batch and size it was made for; any engine of
// the family may step it.
struct b2sd_state {
    uint64_t family = 0;
    int batch = 0, height = 0, width = 0;
    size_t bytes = 0;
    __half* buf = nullptr;
    cudaEvent_t done = nullptr;   // recorded after each step's copy-out; the next step of this stream waits on it
    std::unique_ptr<CondOverride> cond[2];   // the state's own prompt / time block; none: the stepping engine's global values
    // the state's own Canny thresholds (b2sd_state_set_canny_thresholds): host values any engine passes to canny_head
    bool canny = false;   // the family's engines run Canny
    bool canny_own = false;
    double canny_low = 100, canny_high = 200;
};

struct b2sd_engine {
    b2sd_config cfg{};
    int lh = 0, lw = 0;  // latent extents
    std::shared_ptr<WeightStore> ws;
    std::map<std::string, Raw>& raw;
    Arena& weights;
    Arena& raw_only;
    bool& raw_released;
    bool& imported;
    std::map<std::string, __half*>& packed;
    std::map<std::string, float*>& fvec;
    std::map<std::string, size_t>& packed_bytes;
    std::map<std::string, size_t>& fvec_bytes;
    Arena state{16u << 20};      // stream state + small persistent vectors
    Arena prog{512u << 20};      // activations / per-program buffers (reset at prepare)
    explicit b2sd_engine(std::shared_ptr<WeightStore> s)
        : ws(std::move(s)), raw(ws->raw), weights(ws->weights), raw_only(ws->raw_only), raw_released(ws->raw_released),
          imported(ws->imported), packed(ws->packed), fvec(ws->fvec), packed_bytes(ws->packed_bytes), fvec_bytes(ws->fvec_bytes) {}

    // persistent stream state (StreamDiffusion attributes)
    Act x_in;             // UNet input batch: slot 0 = fresh x_t, slots 1.. = x_t_latent_buffer
    __half* noise = nullptr;   // init_noise, NHWC [B][lh][lw][4]
    float* coef = nullptr;     // [4][B]
    float* tsteps = nullptr;   // [B]
    __half* ctx = nullptr;     // prompt embeddings [ctx_tokens][D]
    float* temb_sin = nullptr; // [B][C0]
    float* temb_h = nullptr;   // [B][4*C0]
    float* temb = nullptr;     // [B][4*C0]
    float* cn_temb_h[B2SD_MAX_CONTROLNETS] = {};   // each ControlNet's time_embedding (its own weights), [B][4*C0]
    float* cn_temb[B2SD_MAX_CONTROLNETS] = {};
    // per-slot ControlNet conditioning scales [nets][B] that the zero convs read (net i row i, in the time block), and the
    // engine's global values (1 after b2sd_create)
    float* cn_scale = nullptr;
    float cn_scale_global[B2SD_MAX_CONTROLNETS][16];
    float* gn_ws = nullptr;    // GroupNorm chunk partials (shared: launches are stream-ordered)
    int* tile_counters = nullptr;
    float coef_host[4][64]{};

    __half* ctx_global = nullptr;   // the global prompt embeddings and timesteps: ctx / tsteps again after a state's refresh
    float* tsteps_global = nullptr;
    // IP-Adapter image prompt (cfg.ip_tokens > 0): the image tokens the image program reads, [ATTN_IP_KEYS][D] with zeroed rows
    // past the prompt's tokens, and the global ones; the token count and scale of the global prompt.  The image program writes
    // every UNet cross-attention's image K / V^T and the token count the attention kernel reads (ip_count) into the prompt block.
    __half* ip_tok = nullptr;
    __half* ip_tok_global = nullptr;
    int ip_n_global = 0;
    float ip_scale_global = 1.f;
    float ip_scale = 1.f;   // the scale the image program's V^T launches apply when they run
    int* ip_count = nullptr;

    // The conditioning the frame program reads, as two contiguous blocks: [COND_PROMPT] every cross-attention K / V^T cache
    // (UNet and ControlNet), [COND_TIME] every resnet's per-slot time bias.  A step first makes each block hold what its state
    // is stepped with (the state's override, else this lane's global values), with one copy when it holds something else.
    struct CondBlock {
        char* p = nullptr;        // read by the frame program
        char* global = nullptr;   // this lane's copy of its global values (b2sd_prepare, b2sd_set_prompt_embeds / _timesteps)
        size_t cap = 0, used = 0;
        uint64_t held = 0;        // what p holds: COND_GLOBAL, the id of an override, or COND_UNKNOWN
        void* take(size_t bytes) {
            bytes = (bytes + 1023) & ~size_t(1023);
            if (used + bytes > cap) {
                b2_set_error("conditioning block of %zu bytes exhausted", cap);
                return nullptr;
            }
            void* r = p + used;
            used += bytes;
            return r;
        }
    } cond[2];
    int64_t cond_binds = 0;   // copies into a block by a step (b2sd_conditioning_binds)

    unsigned long long* ln_stats = nullptr;   // slab of per-row LayerNorm statistics [rows][2] (see IgEpilogue::rowstat_out)
    size_t ln_stats_cap = 0, ln_stats_used = 0;   // in 64-bit words
    std::vector<Op> prog_frame, prog_prompt, prog_time, prog_image;
    std::map<std::string, Act> taps;
    SmallConvArgs head{};   // encoder head (reads the caller's frame)
    // each ControlNet's conditioning embedding conv_in (reads the caller's frame as the control image, with processor FRAME)
    SmallConvArgs cn_head[B2SD_MAX_CONTROLNETS]{};
    SmallConvArgs hed_head{};  // HED's first conv (reads the caller's frame) when a control image is its edge map
    // Canny (a net with processor B2SD_CONTROL_CANNY): canny_head (reads the caller's frame) writes canny.cls, stage 1 of the
    // frame program runs the hysteresis launches on it.  The thresholds are host values passed to canny_head when a step
    // launches it: the stepped state's own, else the engine's global ones (b2sd_set_canny_thresholds).
    uint8_t* canny_cls = nullptr;
    CannyCclArgs canny{};
    double canny_low = 100, canny_high = 200;
    struct U8Tap { const uint8_t* p; int h, w, c; };
    std::map<std::string, U8Tap> u8_taps;   // dense u8 [1][h][w][c] buffers, read back as fp16 by b2sd_get_tensor
    int control_processor(int net) const { return net == 0 ? cfg.control_processor : cfg.control_processor_more[net - 1]; }
    bool reads_canny() const {
        for (int i = 0; i < cfg.controlnet; ++i)
            if (control_processor(i) == B2SD_CONTROL_CANNY) return true;
        return false;
    }
    Act image;              // decoder output, fp16 NHWC (ld 8)
    bool built = false;
    int concurrency = 1;   // frames expected in flight on this GPU (b2sd_set_concurrency): > 1 selects the throughput launch policy
    int launches = 0;
    std::string cur;   // name prefix of the layer being built (debug / profiling labels)
    bool allow_swap = false;  // builders enable the swapped GEMM orientation for UNet contractions (never TAESD / V^T / GEGLU)
    // Stepping a stream state (b2sd_step_state): the frame program is cut into [encoder body | last encoder conv + UNet +
    // scheduler step | decoder].  Only the middle stage reads and writes slots 1.. of x_in, so the state is copied in before it
    // and out after it, and steps of one state chain through the state's event.
    size_t idx_enc_end = 0, idx_unet_end = 0;          // stage boundaries inside prog_frame
    // the CUDA graph of each program range run_frame is called with, captured on first use: GRAPH_WHOLE is all of prog_frame
    // (b2sd_step_ex), GRAPH_STAGE + i the i-th stage of a state's step
    enum { GRAPH_WHOLE = 0, GRAPH_STAGE = 1, NUM_GRAPHS = 4 };
    cudaGraphExec_t graph_exec[NUM_GRAPHS] = {};
    void drop_graphs() {
        for (auto& g : graph_exec)
            if (g) { cudaGraphExecDestroy(g); g = nullptr; }
    }

    ~b2sd_engine() { drop_graphs(); }

    // ---- parameters -----------------------------------------------------------------------------
    const Raw* get(const std::string& key) {
        auto it = raw.find(key);
        if (it == raw.end()) {
            b2_set_error("missing weight '%s'", key.c_str());
            return nullptr;
        }
        return &it->second;
    }
    bool has(const std::string& key) const { return raw.count(key) != 0; }

    // fp32 device vector = sum of the named 1-D parameters (optionally row-permuted)
    float* vec(const std::vector<std::string>& keys, const std::vector<int>* perm = nullptr, int pad_to = 0) {
        std::string ck = "v:";
        for (auto& k : keys) ck += k + "+";
        if (perm) ck += "perm";
        auto it = fvec.find(ck);
        if (it != fvec.end()) return it->second;
        std::vector<float> host;
        for (auto& k : keys) {
            const Raw* r = get(k);
            if (!r) return nullptr;
            if (host.empty()) host.assign(r->host.begin(), r->host.end());
            else
                for (size_t i = 0; i < host.size() && i < r->host.size(); ++i) host[i] += r->host[i];
        }
        if (perm) {
            std::vector<float> t(perm->size());
            for (size_t i = 0; i < perm->size(); ++i) t[i] = (*perm)[i] >= 0 ? host[(*perm)[i]] : 0.f;
            host.swap(t);
        }
        if ((int)host.size() < pad_to) host.resize(pad_to, 0.f);
        float* d = static_cast<float*>(weights.alloc(host.size() * sizeof(float)));
        if (!d) return nullptr;
        if (cudaMemcpy(d, host.data(), host.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) return nullptr;
        fvec[ck] = d;
        fvec_bytes[ck] = host.size() * sizeof(float);
        return d;
    }

    // A raw parameter a packing kernel is about to read (its fused value while b2sd_apply_lora rebuilds a cache entry)
    const Raw* pack_source(const std::string& key) {
        const Raw* r = get(key);
        if (r && !r->p) {
            b2_set_error("parameter '%s' was released after the first prepare and is not in the packed cache", key.c_str());
            return nullptr;
        }
        return r;
    }
    // Make a cache entry: record how to rebuild it from its raw parameters (b2sd_apply_lora), then build it once
    int record_rebuild(const std::string& name, std::vector<std::string> keys, std::function<int(cudaStream_t)> fn, cudaStream_t s) {
        WeightStore::Rebuild& rb = ws->rebuild[name];
        rb.keys = std::move(keys);
        rb.fn = std::move(fn);
        return rb.fn(s);
    }

    // fp32 [cin*9][cout] weights of a tiny-Cin conv (cached)
    const float* small_w(const std::string& key, cudaStream_t s) {
        auto it = fvec.find("sw:" + key);
        if (it != fvec.end()) return it->second;
        const Raw* r = pack_source(key);
        if (!r) return nullptr;
        const int cout = (int)r->shape[0], cin = (int)r->shape[1];
        float* d = static_cast<float*>(weights.alloc((size_t)cin * 9 * cout * sizeof(float)));
        WeightStore* w = ws.get();
        if (!d || record_rebuild("sw:" + key, {key}, [=](cudaStream_t st) { return smallconv_prep_launch(w->src(key), d, cout, cin, st); }, s))
            return nullptr;
        fvec["sw:" + key] = d;
        fvec_bytes["sw:" + key] = (size_t)cin * 9 * cout * sizeof(float);
        return d;
    }

    struct ConvSeg { std::string key; int c0, cn, taps; };
    // packed [rows_pad][K] matrix, K = concat of segments each ordered [tap][c]
    __half* pack_conv(const std::string& name, const std::vector<ConvSeg>& segs, int rows, int* k_out,
                      cudaStream_t s) {
        int K = 0;
        for (auto& g : segs) K += g.taps * g.cn;
        *k_out = K;
        auto it = packed.find(name);
        if (it != packed.end()) return it->second;
        const int rows_pad = (rows + 15) / 16 * 16;
        __half* dst = static_cast<__half*>(weights.alloc((size_t)rows_pad * K * 2));
        if (!dst) return nullptr;
        std::vector<std::string> keys;
        std::vector<int> cin_total;
        for (auto& g : segs) {
            const Raw* r = pack_source(g.key);
            if (!r) return nullptr;
            keys.push_back(g.key);
            cin_total.push_back((int)r->shape[1]);
        }
        WeightStore* w = ws.get();
        const size_t bytes = (size_t)rows_pad * K * 2;
        if (record_rebuild(name, keys, [=](cudaStream_t st) {
                if (cudaMemsetAsync(dst, 0, bytes, st) != cudaSuccess) return -1;
                int koff = 0;
                for (size_t i = 0; i < segs.size(); ++i) {
                    const ConvSeg& g = segs[i];
                    if (pack_conv_weight_launch(w->src(g.key), dst, K, koff, rows, cin_total[i], g.taps, g.c0, g.cn, st)) return -1;
                    koff += g.taps * g.cn;
                }
                return 0;
            }, s))
            return nullptr;
        packed[name] = dst;
        packed_bytes[name] = bytes;
        return dst;
    }
    // rows gathered from one or more [*, K] matrices: spec = list of (key, perm).  The gathers of an entry, as a rebuild step.
    std::function<int(cudaStream_t)> gather_fn(const std::vector<std::pair<std::string, std::vector<int>>>& parts, int K,
                                               __half* dst, size_t bytes, cudaStream_t s) {
        std::vector<std::pair<std::string, const int*>> dparts;
        std::vector<int> counts;
        for (auto& p : parts) {
            if (!pack_source(p.first)) return nullptr;
            int* dperm = static_cast<int*>(weights.alloc(p.second.size() * sizeof(int)));
            if (!dperm) return nullptr;
            cudaMemcpyAsync(dperm, p.second.data(), p.second.size() * sizeof(int), cudaMemcpyHostToDevice, s);
            cudaStreamSynchronize(s);  // host vector may die before the copy otherwise
            dparts.emplace_back(p.first, dperm);
            counts.push_back((int)p.second.size());
        }
        WeightStore* w = ws.get();
        return [=](cudaStream_t st) {
            if (cudaMemsetAsync(dst, 0, bytes, st) != cudaSuccess) return -1;
            size_t r0 = 0;
            for (size_t i = 0; i < dparts.size(); ++i) {
                if (gather_rows_launch(w->src(dparts[i].first), K, dparts[i].second, dst + r0 * K, K, counts[i], K, st)) return -1;
                r0 += counts[i];
            }
            return 0;
        };
    }
    static std::vector<std::string> part_keys(const std::vector<std::pair<std::string, std::vector<int>>>& parts) {
        std::vector<std::string> k;
        for (auto& p : parts) k.push_back(p.first);
        return k;
    }
    __half* pack_rows(const std::string& name, const std::vector<std::pair<std::string, std::vector<int>>>& parts,
                      int K, cudaStream_t s) {
        auto it = packed.find(name);
        if (it != packed.end()) return it->second;
        size_t rows = 0;
        for (auto& p : parts) rows += p.second.size();
        const size_t rows_pad = (rows + 15) / 16 * 16;
        __half* dst = static_cast<__half*>(weights.alloc(rows_pad * K * 2));
        if (!dst) return nullptr;
        auto gather = gather_fn(parts, K, dst, rows_pad * K * 2, s);
        if (!gather || record_rebuild(name, part_keys(parts), gather, s)) return nullptr;
        packed[name] = dst;
        packed_bytes[name] = rows_pad * K * 2;
        return dst;
    }

    // LayerNorm folded into a consumer GEMM (IgEpilogue::colsum): W' = gather(parts) diag(gamma) in place of the gathered rows,
    // colsum[n] = sum_k W'[n][k], bias'[n] = sum_k W[n][k] beta[k] + bias[n].  Cached like every packed parameter.
    struct LnFold { __half* w = nullptr; const float* colsum = nullptr; const float* bias = nullptr; };
    int fold_ln(const std::string& name, const std::vector<std::pair<std::string, std::vector<int>>>& parts, int K,
                const std::string& ln_prefix, const float* bias_vec, LnFold* out, cudaStream_t s) {
        size_t rows = 0;
        for (auto& p : parts) rows += p.second.size();
        const size_t rows_pad = (rows + 15) / 16 * 16;
        const bool done = packed.count(name) && fvec.count(name + ":cs") && fvec.count(name + ":b");
        if (!done) {
            // one rebuild step for the three entries: the gathered rows, then the fold on them
            __half* w = static_cast<__half*>(weights.alloc(rows_pad * K * 2));
            if (!w) return -1;
            auto gather = gather_fn(parts, K, w, rows_pad * K * 2, s);
            const float* gamma = vec({ln_prefix + ".weight"});
            const float* beta = vec({ln_prefix + ".bias"});
            float* cs = static_cast<float*>(weights.alloc(rows_pad * sizeof(float)));
            float* bb = static_cast<float*>(weights.alloc(rows_pad * sizeof(float)));
            if (!gather || !gamma || !beta || !cs || !bb) return -1;
            TRY(record_rebuild(name, part_keys(parts), [=](cudaStream_t st) {
                TRY(gather(st));
                if (cudaMemsetAsync(bb, 0, rows_pad * sizeof(float), st) != cudaSuccess) return -1;
                TRY(row_dot_launch(w, (long)rows, K, beta, bias_vec, bb, st));     // on the un-scaled rows
                TRY(scale_cols_launch(w, (long)rows_pad, K, gamma, st));
                return row_sum_launch(w, (long)rows_pad, K, cs, st);
            }, s));
            packed[name] = w; packed_bytes[name] = rows_pad * K * 2;
            fvec[name + ":cs"] = cs; fvec_bytes[name + ":cs"] = rows_pad * sizeof(float);
            fvec[name + ":b"] = bb; fvec_bytes[name + ":b"] = rows_pad * sizeof(float);
        }
        out->w = packed[name];
        out->colsum = fvec[name + ":cs"];
        out->bias = fvec[name + ":b"];
        return 0;
    }
    unsigned long long* alloc_rowstat(long rows) {
        if (ln_stats_used + 2 * (size_t)rows > ln_stats_cap) {
            b2_set_error("LayerNorm statistics slab exhausted");
            return nullptr;
        }
        unsigned long long* p = ln_stats + ln_stats_used;
        ln_stats_used += 2 * (size_t)rows;
        return p;
    }

    // ---- program construction helpers -----------------------------------------------------------
    Act new_act(int n, int h, int w, int c, int ld = 0) {
        Act a;
        a.n = n; a.h = h; a.w = w; a.c = c; a.ld = ld ? ld : c;
        a.p = static_cast<__half*>(prog.alloc((size_t)a.elems() * 2));
        return a;
    }
    static ActView view(const Act& a) { return ActView{a.p, a.n, a.h, a.w, a.c, a.ld}; }
    static ActView tokens(const Act& a) { return ActView{a.p, 1, 1, a.n * a.h * a.w, a.c, a.ld}; }

    // choose N tile / split-K for a good grid (igemm_autotile), plan, and append the launch
    // append a planned contraction
    // scale_src: acc_scale is read from there when the launch runs (the image program's V^T: the scale of the image prompt
    // being computed)
    void push_igemm(std::vector<Op>& dst, const IgemmDesc& d, const IgemmPlan& plan, const std::string& label, double flops,
                    const float* scale_src = nullptr) {
        if (&dst == &prog_frame) launches += 1;
        if (scale_src)
            dst.push_back(Op([plan, sp = scale_src](cudaStream_t s) {
                IgemmPlan q = plan;
                q.p.epi.acc_scale = *sp;
                return igemm_launch(q, s);
            }, label, flops));
        else
            dst.push_back(Op([plan](cudaStream_t s) { return igemm_launch(plan, s); }, label, flops));
        dst.back().rec.kind = B2SD_LAUNCH_IGEMM;
        igemm_record(d, &plan, &dst.back().rec.igemm, &dst.back().rec.plan);
    }

    void push_attn(const AttnPlan& plan, const std::string& label) {
        const AttnDesc& a = plan.d;
        launches += 1;
        prog_frame.push_back(Op([plan](cudaStream_t st) { return attn_launch(plan, st); }, label,
                                4.0 * a.nb * a.heads * (double)a.sq * a.skv * a.d_real));
        b2sd_launch_record& r = prog_frame.back().rec;
        r.kind = B2SD_LAUNCH_ATTN;
        r.attn = b2sd_attn_desc{a.q, a.ldq, a.k, a.ldk, (int64_t)a.k_bstride, (int64_t)a.k_rows, a.vt, a.ldvt, (int64_t)a.vt_bstride,
                                (int64_t)a.vt_cols, a.out, a.ldo, a.nb, a.heads, a.sq, a.skv, a.d_real, a.dp};
        r.attn_k_ip = a.k_ip; r.attn_vt_ip = a.vt_ip; r.attn_n_ip = a.n_ip;
    }

    // choose N tile / split-K for a good grid (igemm_autotile), plan, and append the launch
    int add_igemm(std::vector<Op>& dst, IgemmDesc d, const float* scale_src = nullptr) {
        const bool geglu = (d.epi.flags & IG_GEGLU) != 0;
        const int n_gemm = geglu ? 2 * d.epi.n_valid : d.epi.n_valid;
        const bool extras = d.epi.rowstat_out || d.epi.colsum || d.epi.out2;   // not implemented by the swapped-orientation epilogue
        // several frames in flight: spreading one contraction over fewer K slices costs latency but less SM time (cluster reduction)
        if (concurrency > 1 && d.max_splits == 0) d.max_splits = 4;
        // ... and with the GPU filled by >= 4 frames, CTA pairs without split-K use the least SM time per contraction
        // (igemm_autotile).  Two stage-pipelined lanes of ONE stateful stream (T > 1) run mostly one UNet at a time and keep
        // split-K.
        if (concurrency >= 4 && d.pair_auto == 0) { d.pair_auto = 1; d.pair_splits = 1; }
        IgemmPlan plan;
        TRY(igemm_autotile(d, allow_swap && !extras, &plan));
        if (d.epi.out2 && d.epi.col2 % plan.p.BN != 0) {   // an N tile must be all q/k or all v (igemm_autotile filters on it)
            b2_set_error("fused q/k/v projection: N tile %d does not divide the V offset %d", plan.p.BN, d.epi.col2);
            return -1;
        }
        char label[256];
        snprintf(label, sizeof(label), "igemm %s rows=%ld n=%d kb=%d bn=%d splits=%d grid=%u,%u,%u %s", cur.c_str(),
                 plan.rows_total, d.epi.n_valid, plan.p.total_kb, plan.p.BN, plan.splits, plan.grid.x, plan.grid.y,
                 plan.grid.z, plan.p.swap ? "swapped" : (plan.pair ? "pairs" : "taps"));
        push_igemm(dst, d, plan, label, 2.0 * (double)plan.rows_total * n_gemm * plan.p.total_kb * IG_BK, scale_src);
        return 0;
    }

    int add_groupnorm(const Act& xa, const Act* xb, const std::string& prefix, const Act& y, float eps, int silu) {
        GroupNormArgs a{};
        a.xa = xa.p; a.ca = xa.c; a.lda = xa.ld;
        if (xb) { a.xb = xb->p; a.cb = xb->c; a.ldb = xb->ld; }
        a.gamma = vec({prefix + ".weight"});
        a.beta = vec({prefix + ".bias"});
        if (!a.gamma || !a.beta) return -1;
        a.y = y.p; a.ldy = y.ld;
        a.nb = xa.n; a.hw = xa.h * xa.w; a.groups = cfg.norm_groups; a.eps = eps; a.silu = silu;
        a.partial = gn_ws;
        a.counters = tile_counters;   // zero-initialised, self re-arming
        launches += 1;
        prog_frame.push_back(Op([a](cudaStream_t s) { return groupnorm_launch(a, s); }, "groupnorm " + prefix));
        b2sd_launch_record& r = prog_frame.back().rec;
        r.kind = B2SD_LAUNCH_GROUPNORM;
        r.groupnorm = b2sd_groupnorm_args{a.xa, a.ca, a.lda, a.xb, a.cb, a.ldb, a.gamma, a.beta, a.y, a.ldy, a.nb, a.hw, a.groups,
                                          a.eps, a.silu};
        return 0;
    }

    int add_layernorm(const Act& x, const std::string& prefix, const Act& y) {
        const float* g = vec({prefix + ".weight"});
        const float* b = vec({prefix + ".bias"});
        if (!g || !b) return -1;
        const long rows = (long)x.n * x.h * x.w;
        const __half* xp = x.p; __half* yp = y.p;
        const int ldx = x.ld, ldy = y.ld, c = x.c;
        ++launches;
        prog_frame.push_back(Op([=](cudaStream_t s) { return layernorm_launch(xp, ldx, g, b, yp, ldy, rows, c, 1e-5f, s); }, "layernorm " + prefix));
        b2sd_launch_record& r = prog_frame.back().rec;
        r.kind = B2SD_LAUNCH_LAYERNORM;
        r.layernorm = b2sd_layernorm_args{xp, ldx, g, b, yp, ldy, (int64_t)rows, c, 1e-5f};
        return 0;
    }

    // conv3x3 (or 1x1) over one source with bias / relu / residual
    int add_conv(std::vector<Op>& dst, const Act& x, const std::string& wkey, const std::string& bkey, int taps,
                 int stride, const Act& y, int flags, const Act* res, cudaStream_t s, float acc_scale = 1.f,
                 float res_scale = 1.f, const float* acc_scale_b = nullptr) {
        const Raw* w = get(wkey);
        if (!w) return -1;
        cur = wkey;
        const int cout = (int)w->shape[0];
        int K = 0;
        __half* wp = pack_conv(wkey, {{wkey, 0, x.c, taps}}, cout, &K, s);
        if (!wp) return -1;
        IgemmDesc d{};
        d.nseg = 1; d.src[0] = view(x); d.ntap[0] = taps;
        d.w = wp; d.w_rows = (cout + 15) / 16 * 16; d.w_ld = K;
        d.stride = stride;
        d.Nb = y.n; d.Ho = y.h; d.Wo = y.w;
        d.epi.out = y.p; d.epi.ldc = y.ld;
        if (!bkey.empty()) {
            d.epi.colbias = vec({bkey}, nullptr, 16);
            if (!d.epi.colbias) return -1;
        }
        d.epi.colbias_bstride = 0;
        if (res) { d.epi.res = res->p; d.epi.ldr = res->ld; }
        d.epi.acc_scale = acc_scale; d.epi.res_scale = res_scale;
        d.epi.acc_scale_b = acc_scale_b;
        d.epi.flags = flags;
        d.epi.n_valid = cout;
        // the TAESD body at 256x256 and above: persistent halo-tile kernel with resident weights (tconv.cu)
        static const bool no_tconv = getenv("B2_NO_TCONV") != nullptr;
        static const char* tc_min = getenv("B2_TCONV_MIN_TILES");
        const long tiles = (long)y.n * ((y.h + TC_TH - 1) / TC_TH) * ((y.w + TC_TW - 1) / TC_TW);
        if (!no_tconv && stride == 1 && tconv_eligible(d) && tiles >= (tc_min ? atoi(tc_min) : 2 * IG_SMS)) {
            TconvPlan tp;
            TRY(tconv_plan(d, &tp));
            char label[256];
            snprintf(label, sizeof(label), "tconv %s rows=%ld tiles=%d grid=%u nbuf=%d", wkey.c_str(), tp.rows_total, tp.p.num_tiles,
                     tp.grid.x, tp.p.nbuf);
            if (&dst == &prog_frame) launches += 1;
            dst.push_back(Op([tp](cudaStream_t st) { return tconv_launch(tp, st); }, label, 2.0 * (double)tp.rows_total * cout * K));
            dst.back().rec.kind = B2SD_LAUNCH_TCONV;
            igemm_record(d, nullptr, &dst.back().rec.igemm, &dst.back().rec.plan);
            return 0;
        }
        return add_igemm(dst, d);
    }

    // Linear over tokens: y = x W^T (+bias) (+res)
    struct LinExtra {   // LayerNorm-fold / row-statistics / transposed-V options of a Linear (IgEpilogue)
        unsigned long long* rowstat_out = nullptr;
        const unsigned long long* rowstat_in = nullptr;
        const float* colsum = nullptr;
        int ln_c = 0;
        __half* out2 = nullptr;
        int ld2 = 0, col2 = 0;
    };
    int add_linear(std::vector<Op>& dst, const ActView& x, const __half* w, int n, int k, const float* bias,
                   __half* out, int ldc, const __half* res, int ldr, int flags = 0, int n_valid = -1,
                   const LinExtra* ex = nullptr) {
        IgemmDesc d{};
        if (ex) {
            d.epi.rowstat_out = ex->rowstat_out;
            d.epi.rowstat_in = ex->rowstat_in;
            d.epi.colsum = ex->colsum;
            d.epi.ln_inv_c = ex->ln_c ? 1.f / (float)ex->ln_c : 0.f;
            d.epi.ln_eps = 1e-5f;
            d.epi.out2 = ex->out2; d.epi.ld2 = ex->ld2; d.epi.col2 = ex->col2;
        }
        d.nseg = 1; d.src[0] = x; d.ntap[0] = 1;
        d.w = w; d.w_rows = n; d.w_ld = k;
        d.stride = 1;
        d.Nb = 1; d.Ho = 1; d.Wo = x.W;
        d.epi.out = out; d.epi.ldc = ldc;
        d.epi.colbias = bias; d.epi.colbias_bstride = 0;
        d.epi.res = res; d.epi.ldr = ldr;
        d.epi.acc_scale = 1.f; d.epi.res_scale = 1.f;
        d.epi.flags = flags;
        d.epi.n_valid = n_valid >= 0 ? n_valid : n;
        return add_igemm(dst, d);
    }

    int build_resnet(const std::string& p, const Act& xa, const Act* xb, int cout, const float* emb, Act* out, cudaStream_t s,
                     float eps = 1e-5f);
    int build_vae_attention(const std::string& p, const Act& x, Act* out, cudaStream_t s);
    int build_kl_encoder(Act* out, std::string* latent_conv, cudaStream_t s);
    int build_kl_decoder(const Act& x0, cudaStream_t s);
    std::vector<float> host_copy(const std::string& key);
    int derive(const std::string& name, const std::vector<int64_t>& shape, const std::vector<float>& v);
    const float* const_vec(const std::string& name, const std::vector<float>& v);
    int build_cond_embedding(int net, const uint8_t** shared_control, Act* out, cudaStream_t s);
    int build_hed(const uint8_t** control, cudaStream_t s);
    int build_canny(const uint8_t** control, cudaStream_t s);
    int build_controlnet(int net, const Act& cond, std::vector<Act>& skips, Act* mid, cudaStream_t s);
    int build_transformer(const std::string& p, const Act& x, int heads, Act* out, cudaStream_t s);
    int build_taesd_block(const std::string& p, const Act& x, Act* out, cudaStream_t s);
    int build_program(cudaStream_t s);
    // ops[a, b) on s
    int run(std::vector<Op>& ops, cudaStream_t s, size_t a = 0, size_t b = SIZE_MAX) {
        static const bool dbg = getenv("B200SD_DEBUG_SYNC") != nullptr;
        static const char* skip = getenv("B200SD_SKIP");  // debug: "groupnorm,attn" drops those launches (timing only)
        static const char* skip_name = getenv("B200SD_SKIP_NAME");  // debug: drop launches whose label contains this substring
        for (size_t idx = a; idx < b && idx < ops.size(); ++idx) {
            Op& op = ops[idx];
            if (skip) {
                const std::string kind = op.name.substr(0, op.name.find(' '));
                if (!kind.empty() && std::string(skip).find(kind) != std::string::npos) continue;
            }
            if (skip_name && op.name.find(skip_name) != std::string::npos) continue;
            TRY(op(s));
            if (dbg) {
                cudaError_t e = cudaStreamSynchronize(s);
                if (e != cudaSuccess) {
                    b2_set_error("op %zu '%s' failed: %s", idx, op.name.c_str(), cudaGetErrorString(e));
                    fprintf(stderr, "b2sd: op %zu '%s' failed: %s\n", idx, op.name.c_str(), cudaGetErrorString(e));
                    return -1;
                }
            }
        }
        return 0;
    }
};

// ------------------------------------------------------------------------------------------------
// ResnetBlock2D (diffusers resnet.py): GN+SiLU -> conv1 (+temb) -> GN+SiLU -> conv2, + shortcut(x).  emb = nullptr: no time
// embedding (the AutoencoderKL's resnets, temb_channels=None).
int b2sd_engine::build_resnet(const std::string& p, const Act& xa, const Act* xb, int cout, const float* emb, Act* out,
                              cudaStream_t s, float eps) {
    cur = p;
    allow_swap = true;
    const int cin = xa.c + (xb ? xb->c : 0);
    const int B = xa.n;
    Act n1 = new_act(B, xa.h, xa.w, cin);
    TRY(add_groupnorm(xa, xb, p + "norm1", n1, eps, 1));
    // conv1 with per-sample column bias = conv1.bias + time_emb_proj(silu(emb))
    Act h1 = new_act(B, xa.h, xa.w, cout);
    {
        int K = 0;
        __half* wp = pack_conv(p + "conv1.weight", {{p + "conv1.weight", 0, cin, 9}}, cout, &K, s);
        if (!wp) return -1;
        const float* colbias = nullptr;
        if (emb) {
            float* cb = static_cast<float*>(cond[COND_TIME].take((size_t)B * cout * sizeof(float)));
            const float* bsum = vec({p + "conv1.bias", p + "time_emb_proj.bias"});
            const Raw* wt = get(p + "time_emb_proj.weight");
            if (!cb || !bsum || !wt) return -1;
            const int tdim = (int)wt->shape[1];
            const __half* wtp = wt->p;
            prog_time.push_back(Op([=](cudaStream_t st) { return small_linear_launch(emb, tdim, wtp, bsum, cb, cout, B, cout, tdim, 1, st); }, "temb " + p,
                                   small_linear_record(emb, tdim, wtp, bsum, cb, cout, B, cout, tdim, 1)));
            colbias = cb;
        } else {
            colbias = vec({p + "conv1.bias"}, nullptr, 16);
            if (!colbias) return -1;
        }
        IgemmDesc d{};
        d.nseg = 1; d.src[0] = view(n1); d.ntap[0] = 9;
        d.w = wp; d.w_rows = cout; d.w_ld = K; d.stride = 1;
        d.Nb = B; d.Ho = xa.h; d.Wo = xa.w;
        d.epi.out = h1.p; d.epi.ldc = h1.ld;
        d.epi.colbias = colbias; d.epi.colbias_bstride = emb ? cout : 0;
        d.epi.acc_scale = 1.f; d.epi.res_scale = 1.f; d.epi.n_valid = cout;
        TRY(add_igemm(prog_frame, d));
    }
    Act n2 = new_act(B, xa.h, xa.w, cout);
    TRY(add_groupnorm(h1, nullptr, p + "norm2", n2, eps, 1));
    *out = new_act(B, xa.h, xa.w, cout);
    IgemmDesc d{};
    d.stride = 1; d.Nb = B; d.Ho = xa.h; d.Wo = xa.w;
    d.epi.out = out->p; d.epi.ldc = out->ld;
    d.epi.acc_scale = 1.f; d.epi.res_scale = 1.f; d.epi.n_valid = cout;
    d.src[0] = view(n2); d.ntap[0] = 9;
    int K = 0;
    if (has(p + "conv_shortcut.weight")) {
        // out = conv2(n2) + conv_shortcut(cat[xa, xb]): one K loop over three TMA sources
        std::vector<ConvSeg> segs = {{p + "conv2.weight", 0, cout, 9}, {p + "conv_shortcut.weight", 0, xa.c, 1}};
        d.nseg = 2; d.src[1] = view(xa); d.ntap[1] = 1;
        if (xb) {
            segs.push_back({p + "conv_shortcut.weight", xa.c, xb->c, 1});
            d.nseg = 3; d.src[2] = view(*xb); d.ntap[2] = 1;
        }
        __half* wp = pack_conv(p + "conv2+shortcut", segs, cout, &K, s);
        if (!wp) return -1;
        d.w = wp; d.w_rows = cout; d.w_ld = K;
        d.epi.colbias = vec({p + "conv2.bias", p + "conv_shortcut.bias"});
    } else {
        if (xb) {
            b2_set_error("resnet %s: concat input without conv_shortcut", p.c_str());
            return -1;
        }
        __half* wp = pack_conv(p + "conv2.weight", {{p + "conv2.weight", 0, cout, 9}}, cout, &K, s);
        if (!wp) return -1;
        d.nseg = 1;
        d.w = wp; d.w_rows = cout; d.w_ld = K;
        d.epi.colbias = vec({p + "conv2.bias"});
        d.epi.res = xa.p; d.epi.ldr = xa.ld;
    }
    if (!d.epi.colbias) return -1;
    return add_igemm(prog_frame, d);
}

// Transformer2DModel + BasicTransformerBlock (diffusers transformer_2d.py / attention.py)
int b2sd_engine::build_transformer(const std::string& p, const Act& x, int heads, Act* out, cudaStream_t s) {
    cur = p;
    allow_swap = true;
    const int B = x.n, C = x.c, HW = x.h * x.w;
    const long M = (long)B * HW;
    const int d_real = C / heads;
    const int dp = d_real <= 64 ? 64 : (d_real <= 128 ? 128 : 192);
    const int Cp = heads * dp;
    const int D = cfg.cross_attention_dim, L = cfg.ctx_tokens;
    const std::string t = p + "transformer_blocks.0.";
    auto head_perm = [&](int base) {  // packed row (h*dp+i) <- source row (h*d+i), -1 = zero padding
        std::vector<int> pm(Cp);
        for (int hh = 0; hh < heads; ++hh)
            for (int i = 0; i < dp; ++i) pm[hh * dp + i] = i < d_real ? base + hh * d_real + i : -1;
        return pm;
    };
    Act n = new_act(B, x.h, x.w, C);
    TRY(add_groupnorm(x, nullptr, p + "norm", n, 1e-6f, 0));
    const int HWp = (HW + 7) / 8 * 8;
    const bool one_gemm = (HW % 8 == 0) || B == 1;   // V^T of all batch items is one [Cp][B*HW] matrix (TMA needs 16-byte column origins)
    // LayerNorm folding + fused q/k/v projection: norm1/2/3 never run as kernels.  Each LayerNorm input is produced by a Linear
    // whose epilogue also accumulates the row statistics (rowstat_out); the consumer GEMM runs on the RAW rows with gamma folded
    // into its weights and applies mean / rstd in its epilogue (IgEpilogue::colsum).  B2_NO_LNFOLD=1 restores the three
    // layernorm launches + separate V^T GEMM (also used when the batch's V^T columns need per-image padding).
    static const bool no_fold = getenv("B2_NO_LNFOLD") != nullptr;
    static const char* fold_rows_env = getenv("B2_LNFOLD_MAX_ROWS");   // tuning: disable the fold above this many tokens
    const long fold_max_rows = fold_rows_env ? atol(fold_rows_env) : (1l << 40);
    const bool fold = !no_fold && one_gemm && (long)B * (cfg.height / 8) * (cfg.width / 8) <= fold_max_rows;
    const int inner = 4 * C;
    std::vector<int> gperm;   // GEGLU: weight rows interleaved per 128-wide tile as [64 value | 64 gate]
    {
        const int half = 64;
        for (int tI = 0; tI < inner / half; ++tI) {
            for (int i = 0; i < half; ++i) gperm.push_back(tI * half + i);
            for (int i = 0; i < half; ++i) gperm.push_back(inner + tI * half + i);
        }
    }
    const float* bff1 = vec({t + "ff.net.0.proj.bias"}, &gperm);
    if (!bff1) return -1;
    // proj_in: Linear (SD-Turbo) or 1x1 conv (SD-1.5) -- the same GEMM on NHWC tokens
    const Raw* wpi = get(p + "proj_in.weight");
    if (!wpi) return -1;
    Act hs = new_act(B, x.h, x.w, C);
    unsigned long long *st1 = nullptr, *st2 = nullptr, *st3 = nullptr;
    if (fold) {
        st1 = alloc_rowstat(M); st2 = alloc_rowstat(M); st3 = alloc_rowstat(M);
        if (!st1 || !st2 || !st3) return -1;
    }
    {
        LinExtra ex; ex.rowstat_out = st1;
        TRY(add_linear(prog_frame, tokens(n), wpi->p, C, C, vec({p + "proj_in.bias"}), hs.p, C, nullptr, 0, 0, -1, &ex));
    }
    // ---- self attention
    Act qk = new_act(1, 1, (int)M, 2 * Cp);
    const long vt_ld = one_gemm ? (M + 7) / 8 * 8 : (long)B * HWp;
    const long vt_bstride = one_gemm ? HW : HWp;
    __half* vt = static_cast<__half*>(prog.alloc((size_t)Cp * vt_ld * 2));
    if (!vt) return -1;
    cudaMemsetAsync(vt, 0, (size_t)Cp * vt_ld * 2, s);  // pad columns must stay finite (0 * NaN = NaN in P.V)
    if (fold) {
        // one GEMM: [q | k | v] rows; q/k columns go to `qk`, the V block is stored transposed (K-major V^T for the P.V MMA)
        LnFold f;
        TRY(fold_ln(t + "attn1.qkv+ln", {{t + "attn1.to_q.weight", head_perm(0)}, {t + "attn1.to_k.weight", head_perm(0)},
                                         {t + "attn1.to_v.weight", head_perm(0)}}, C, t + "norm1", nullptr, &f, s));
        LinExtra ex; ex.rowstat_in = st1; ex.colsum = f.colsum; ex.ln_c = C; ex.out2 = vt; ex.ld2 = (int)vt_ld; ex.col2 = 2 * Cp;
        TRY(add_linear(prog_frame, tokens(hs), f.w, 3 * Cp, C, f.bias, qk.p, 2 * Cp, nullptr, 0, 0, -1, &ex));
    } else {
        Act ln = new_act(B, x.h, x.w, C);
        TRY(add_layernorm(hs, t + "norm1", ln));
        __half* wqk = pack_rows(t + "attn1.qk", {{t + "attn1.to_q.weight", head_perm(0)}, {t + "attn1.to_k.weight", head_perm(0)}}, C, s);
        __half* wv = pack_rows(t + "attn1.v", {{t + "attn1.to_v.weight", head_perm(0)}}, C, s);
        if (!wqk || !wv) return -1;
        TRY(add_linear(prog_frame, tokens(ln), wqk, 2 * Cp, C, nullptr, qk.p, 2 * Cp, nullptr, 0));
        // V^T = Wv . ln^T : weights on the M side, tokens on the N side.  TMA needs the per-batch column origin
        // 16-byte aligned, so when HW is not a multiple of 8 each batch item gets its own padded column range.
        allow_swap = false;  // V^T already has the weights on the M side
        for (int bi = 0; bi < (one_gemm ? 1 : B); ++bi) {
            ActView wv_view{wv, 1, 1, Cp, C, C};
            IgemmDesc d{};
            d.nseg = 1; d.src[0] = wv_view; d.ntap[0] = 1;
            d.w = one_gemm ? ln.p : ln.p + (long)bi * HW * ln.ld;
            d.w_rows = one_gemm ? (int)M : HW; d.w_ld = C; d.stride = 1;
            d.Nb = 1; d.Ho = 1; d.Wo = Cp;
            d.epi.out = one_gemm ? vt : vt + (long)bi * HWp;
            d.epi.ldc = (int)vt_ld; d.epi.acc_scale = 1.f; d.epi.res_scale = 1.f;
            d.epi.n_valid = one_gemm ? (int)M : HW;
            TRY(add_igemm(prog_frame, d));
        }
        allow_swap = true;
    }
    Act ao = new_act(B, x.h, x.w, C);
    {
        AttnDesc a{};
        a.q = qk.p; a.ldq = 2 * Cp;
        a.k = qk.p + Cp; a.ldk = 2 * Cp; a.k_bstride = HW; a.k_rows = M;
        a.vt = vt; a.ldvt = (int)vt_ld; a.vt_bstride = vt_bstride; a.vt_cols = one_gemm ? M : (long)B * HWp;
        a.out = ao.p; a.ldo = C;
        a.nb = B; a.heads = heads; a.sq = HW; a.skv = HW; a.d_real = d_real; a.dp = dp;
        AttnPlan plan;
        TRY(attn_plan(a, &plan));
        push_attn(plan, "attn " + p);
    }
    const Raw* wo1 = get(t + "attn1.to_out.0.weight");
    if (!wo1) return -1;
    Act hs2 = new_act(B, x.h, x.w, C);
    {
        LinExtra ex; ex.rowstat_out = st2;
        TRY(add_linear(prog_frame, tokens(ao), wo1->p, C, C, vec({t + "attn1.to_out.0.bias"}), hs2.p, C, hs.p, C, 0, -1, &ex));
    }
    // ---- cross attention against the cached prompt K / V^T
    __half* wk2 = pack_rows(t + "attn2.k", {{t + "attn2.to_k.weight", head_perm(0)}}, D, s);
    __half* wv2 = pack_rows(t + "attn2.v", {{t + "attn2.to_v.weight", head_perm(0)}}, D, s);
    if (!wk2 || !wv2) return -1;
    __half* kc = static_cast<__half*>(cond[COND_PROMPT].take((size_t)L * Cp * 2));
    const int Lpad = 128 * ((L + 127) / 128);
    __half* vct = static_cast<__half*>(cond[COND_PROMPT].take((size_t)Cp * Lpad * 2));
    if (!kc || !vct) return -1;
    {
        allow_swap = false;
        ActView ctxv{ctx, 1, 1, L, D, D};
        TRY(add_linear(prog_prompt, ctxv, wk2, Cp, D, nullptr, kc, Cp, nullptr, 0));
        ActView wvv{wv2, 1, 1, Cp, D, D};
        IgemmDesc d{};
        d.nseg = 1; d.src[0] = wvv; d.ntap[0] = 1;
        d.w = ctx; d.w_rows = L; d.w_ld = D; d.stride = 1;
        d.Nb = 1; d.Ho = 1; d.Wo = Cp;
        d.epi.out = vct; d.epi.ldc = Lpad; d.epi.acc_scale = 1.f; d.epi.res_scale = 1.f; d.epi.n_valid = L;
        TRY(add_igemm(prog_prompt, d));
        allow_swap = true;
    }
    // ---- IP-Adapter: the image tokens' K [64][Cp] and scale * V^T [Cp][64] (UNet only: the ControlNet's stay text-only, as in
    // diffusers).  Rows / columns past the prompt's tokens come from its zeroed token rows, so they are finite.
    __half *kip = nullptr, *vipt = nullptr;
    if (cfg.ip_tokens && p.compare(0, 10, "controlnet") != 0) {   // not under any net's "controlnet." / "controlnet<i>."
        __half* wk = pack_rows(t + "attn2.k_ip", {{t + "attn2.to_k_ip.weight", head_perm(0)}}, D, s);
        __half* wv = pack_rows(t + "attn2.v_ip", {{t + "attn2.to_v_ip.weight", head_perm(0)}}, D, s);
        kip = static_cast<__half*>(cond[COND_PROMPT].take((size_t)ATTN_IP_KEYS * Cp * 2));
        vipt = static_cast<__half*>(cond[COND_PROMPT].take((size_t)Cp * ATTN_IP_KEYS * 2));
        if (!wk || !wv || !kip || !vipt) return -1;
        allow_swap = false;
        ActView tokv{ip_tok, 1, 1, ATTN_IP_KEYS, D, D};
        TRY(add_linear(prog_image, tokv, wk, Cp, D, nullptr, kip, Cp, nullptr, 0));
        ActView wvv{wv, 1, 1, Cp, D, D};
        IgemmDesc d{};
        d.nseg = 1; d.src[0] = wvv; d.ntap[0] = 1;
        d.w = ip_tok; d.w_rows = ATTN_IP_KEYS; d.w_ld = D; d.stride = 1;
        d.Nb = 1; d.Ho = 1; d.Wo = Cp;
        d.epi.out = vipt; d.epi.ldc = ATTN_IP_KEYS; d.epi.acc_scale = 1.f; d.epi.res_scale = 1.f; d.epi.n_valid = ATTN_IP_KEYS;
        TRY(add_igemm(prog_image, d, &ip_scale));
        allow_swap = true;
    }
    Act q2 = new_act(1, 1, (int)M, Cp);
    if (fold) {
        LnFold f;
        TRY(fold_ln(t + "attn2.q+ln", {{t + "attn2.to_q.weight", head_perm(0)}}, C, t + "norm2", nullptr, &f, s));
        LinExtra ex; ex.rowstat_in = st2; ex.colsum = f.colsum; ex.ln_c = C;
        TRY(add_linear(prog_frame, tokens(hs2), f.w, Cp, C, f.bias, q2.p, Cp, nullptr, 0, 0, -1, &ex));
    } else {
        Act ln2 = new_act(B, x.h, x.w, C);
        TRY(add_layernorm(hs2, t + "norm2", ln2));
        __half* wq2 = pack_rows(t + "attn2.q", {{t + "attn2.to_q.weight", head_perm(0)}}, C, s);
        if (!wq2) return -1;
        TRY(add_linear(prog_frame, tokens(ln2), wq2, Cp, C, nullptr, q2.p, Cp, nullptr, 0));
    }
    Act ao2 = new_act(B, x.h, x.w, C);
    {
        AttnDesc a{};
        a.q = q2.p; a.ldq = Cp;
        a.k = kc; a.ldk = Cp; a.k_bstride = 0; a.k_rows = L;
        a.vt = vct; a.ldvt = Lpad; a.vt_bstride = 0; a.vt_cols = L;
        a.out = ao2.p; a.ldo = C;
        a.nb = B; a.heads = heads; a.sq = HW; a.skv = L; a.d_real = d_real; a.dp = dp;
        if (kip) { a.k_ip = kip; a.vt_ip = vipt; a.n_ip = ip_count; }
        AttnPlan plan;
        TRY(attn_plan(a, &plan));
        push_attn(plan, "attn " + p);
    }
    const Raw* wo2 = get(t + "attn2.to_out.0.weight");
    if (!wo2) return -1;
    Act hs3 = new_act(B, x.h, x.w, C);
    {
        LinExtra ex; ex.rowstat_out = st3;
        TRY(add_linear(prog_frame, tokens(ao2), wo2->p, C, C, vec({t + "attn2.to_out.0.bias"}), hs3.p, C, hs2.p, C, 0, -1, &ex));
    }
    // ---- GEGLU feed-forward
    Act ff = new_act(1, 1, (int)M, inner);
    {
        IgemmDesc d{};
        d.nseg = 1; d.ntap[0] = 1;
        d.w_rows = 2 * inner; d.w_ld = C; d.stride = 1;
        d.Nb = 1; d.Ho = 1; d.Wo = (int)M;
        d.BN = 128;   // the 128-column value/gate interleave of the packed rows
        d.epi.out = ff.p; d.epi.ldc = inner; d.epi.acc_scale = 1.f; d.epi.res_scale = 1.f;
        d.epi.flags = IG_GEGLU; d.epi.n_valid = inner;
        if (fold) {
            LnFold f;
            TRY(fold_ln(t + "ff1+ln", {{t + "ff.net.0.proj.weight", gperm}}, C, t + "norm3", bff1, &f, s));
            d.src[0] = tokens(hs3);
            d.w = f.w; d.epi.colbias = f.bias;
            d.epi.rowstat_in = st3; d.epi.colsum = f.colsum; d.epi.ln_inv_c = 1.f / (float)C; d.epi.ln_eps = 1e-5f;
        } else {
            Act ln3 = new_act(B, x.h, x.w, C);
            TRY(add_layernorm(hs3, t + "norm3", ln3));
            __half* wff1 = pack_rows(t + "ff1", {{t + "ff.net.0.proj.weight", gperm}}, C, s);
            if (!wff1) return -1;
            d.src[0] = tokens(ln3);
            d.w = wff1; d.epi.colbias = bff1;
        }
        IgemmPlan plan;
        TRY(igemm_plan(d, &plan));
        push_igemm(prog_frame, d, plan, "igemm geglu " + p, 2.0 * (double)M * (2.0 * inner) * C);
    }
    const Raw* wff2 = get(t + "ff.net.2.weight");
    if (!wff2) return -1;
    Act hs4 = new_act(B, x.h, x.w, C);
    TRY(add_linear(prog_frame, tokens(ff), wff2->p, C, inner, vec({t + "ff.net.2.bias"}), hs4.p, C, hs3.p, C));
    // proj_out + residual with the block input
    const Raw* wpo = get(p + "proj_out.weight");
    if (!wpo) return -1;
    *out = new_act(B, x.h, x.w, C);
    return add_linear(prog_frame, tokens(hs4), wpo->p, C, C, vec({p + "proj_out.bias"}), out->p, C, x.p, x.ld);
}

// AutoencoderTinyBlock: relu(conv(relu(conv(relu(conv(x))))) + x)
int b2sd_engine::build_taesd_block(const std::string& p, const Act& x, Act* out, cudaStream_t s) {
    cur = p;
    allow_swap = false;
    Act a = new_act(x.n, x.h, x.w, x.c), b = new_act(x.n, x.h, x.w, x.c);
    *out = new_act(x.n, x.h, x.w, x.c);
    TRY(add_conv(prog_frame, x, p + ".conv.0.weight", p + ".conv.0.bias", 9, 1, a, IG_RELU, nullptr, s));
    TRY(add_conv(prog_frame, a, p + ".conv.2.weight", p + ".conv.2.bias", 9, 1, b, IG_RELU, nullptr, s));
    return add_conv(prog_frame, b, p + ".conv.4.weight", p + ".conv.4.bias", 9, 1, *out, IG_RELU, &x, s);
}

// The weight prefix of ControlNet `net`: "controlnet." for net 0, "controlnet<i>." for net i (never "controlnet.<i>.", so that
// a key under "controlnet." always belongs to net 0)
static std::string cn_prefix(int net) { return net == 0 ? std::string("controlnet.") : "controlnet" + std::to_string(net) + "."; }

// ControlNetConditioningEmbedding (diffusers controlnet.py): conv_in 3->16 + SiLU, six 3x3 convs 16->16, 16->32/2, 32->32,
// 32->96/2, 96->96, 96->256/2 each + SiLU, conv_out 256->C0.  conv_in reads the caller's frame (b2sd_step_ex launches cn_head
// next to the encoder head); the rest is stage 1 of the frame program (it depends on the frame only).  The 16/32/96-channel
// activations are stored 64/64/128 wide with zero padding columns, so the following layers run as 64/64/128-channel
// tensor-core contractions (zero weights on the padding channels, pack_conv_weight_launch).  The epilogues write only the
// valid columns: the padding is cleared once here, and stays finite (0 * NaN would be NaN).  With several nets each has its
// own; HED and Canny each run once, for the first net that reads their edge map (shared_control[processor], null until then),
// and later ones share it.
int b2sd_engine::build_cond_embedding(int net, const uint8_t** shared_control, Act* out, cudaStream_t s) {
    const std::string p = cn_prefix(net) + "controlnet_cond_embedding.";
    SmallConvArgs& cn_head = this->cn_head[net];
    cur = p;
    allow_swap = false;
    auto padded = [&](int n, int hh, int ww, int c) {
        Act a = new_act(n, hh, ww, c, (c + 63) / 64 * 64);
        if (a.p && a.ld != c && cudaMemsetAsync(a.p, 0, (size_t)a.elems() * 2, s) != cudaSuccess) a.p = nullptr;
        return a;
    };
    Act a = padded(1, cfg.height, cfg.width, 16);
    if (!a.p) { b2_set_error("controlnet: activation allocation failed"); return -1; }
    cn_head = SmallConvArgs{};
    cn_head.wt = small_w(p + "conv_in.weight", s);
    cn_head.bias = vec({p + "conv_in.bias"});
    if (!cn_head.wt || !cn_head.bias) return -1;
    cn_head.y = a.p; cn_head.ldy = a.ld; cn_head.nb = 1; cn_head.h = a.h; cn_head.w_ = a.w; cn_head.cin = 3; cn_head.cout = 16;
    ++launches;
    const int proc = control_processor(net);
    if (proc != B2SD_CONTROL_FRAME) {   // the control image is HED's or Canny's edge map, computed in this stage
        const uint8_t** edge = &shared_control[proc];
        if (!*edge) TRY(proc == B2SD_CONTROL_HED ? build_hed(edge, s) : build_canny(edge, s));
        SmallConvArgs c = cn_head;
        c.x = *edge; c.in_h = a.h; c.in_w = a.w; c.flags = SC_IN_U8 | SC_OUT_SILU;
        prog_frame.push_back(Op([c](cudaStream_t st) { return smallconv_launch(c, st); }, "smallconv controlnet_cond_embedding.conv_in",
                                smallconv_record(c)));
    }
    static const int cout[6] = {16, 32, 32, 96, 96, 256}, stride[6] = {1, 2, 1, 2, 1, 2};
    for (int k = 0; k < 6; ++k) {
        Act x = a;
        x.c = x.ld;   // padding channels enter the contraction (zero activations times zero weights)
        a = padded(1, x.h / stride[k], x.w / stride[k], cout[k]);
        if (!a.p) { b2_set_error("controlnet: activation allocation failed"); return -1; }
        const std::string w = p + "blocks." + std::to_string(k);
        TRY(add_conv(prog_frame, x, w + ".weight", w + ".bias", 9, stride[k], a, IG_SILU, nullptr, s));
    }
    *out = new_act(1, lh, lw, cfg.block_out_channels[0]);
    TRY(add_conv(prog_frame, a, p + "conv_out.weight", p + "conv_out.bias", 9, 1, *out, 0, nullptr, s));
    taps["cn" + std::to_string(net) + "_cond"] = *out;
    if (net == 0) taps["cn_cond"] = *out;
    return 0;
}

// ControlNetHED_Apache2 (controlnet_aux) + HEDdetector's post-processing, at the engine's resolution: h = frame(0..255) - norm;
// five blocks of 3x3 convs + ReLU (3->64 x2, 64->128 x2, 128->256 x3, 256->512 x3, 512->512 x3), blocks 2-5 after a 2x2/2
// max-pool; each block's 1x1 projection to one channel; the five maps upsampled bilinearly, averaged, sigmoid, * 255,
// truncated to the u8 edge image (3 channels).  The first conv reads the caller's frame (hed_head, launched by b2sd_step_ex).
int b2sd_engine::build_hed(const uint8_t** control, cudaStream_t s) {
    const int H = cfg.height, W = cfg.width;
    static const int ch[5] = {64, 128, 256, 512, 512}, nconv[5] = {2, 2, 3, 3, 3};
    cur = "hed";
    allow_swap = false;
    Act a = new_act(1, H, W, ch[0]);
    hed_head = SmallConvArgs{};
    hed_head.wt = small_w("hed.block1.convs.0.weight", s);
    hed_head.bias = vec({"hed.block1.convs.0.bias"});
    hed_head.in_off = vec({"hed.norm"});
    if (!a.p || !hed_head.wt || !hed_head.bias || !hed_head.in_off) return -1;
    hed_head.y = a.p; hed_head.ldy = a.ld; hed_head.nb = 1; hed_head.h = H; hed_head.w_ = W; hed_head.cin = 3; hed_head.cout = ch[0];
    ++launches;
    HedFuseArgs f{};
    for (int b = 0; b < 5; ++b) {
        const std::string p = "hed.block" + std::to_string(b + 1) + ".";
        if (b > 0) {
            Act o = new_act(1, a.h / 2, a.w / 2, a.c);
            if (!o.p) return -1;
            const Act x = a;
            ++launches;
            b2sd_launch_record r{};
            r.kind = B2SD_LAUNCH_MAXPOOL2X2;
            r.maxpool2x2 = b2sd_maxpool2x2_args{x.p, o.p, 1, x.h, x.w, x.c};
            prog_frame.push_back(Op([x, o](cudaStream_t st) { return maxpool2x2_launch(x.p, o.p, 1, x.h, x.w, x.c, st); }, "maxpool2x2 " + p, r));
            a = o;
        }
        for (int k = b == 0 ? 1 : 0; k < nconv[b]; ++k) {
            Act o = new_act(1, a.h, a.w, ch[b]);
            const std::string w = p + "convs." + std::to_string(k);
            TRY(add_conv(prog_frame, a, w + ".weight", w + ".bias", 9, 1, o, IG_RELU, nullptr, s));
            a = o;
        }
        float* m = static_cast<float*>(prog.alloc((size_t)a.h * a.w * sizeof(float)));
        const float* pw = vec({p + "projection.weight"});
        const float* pb = vec({p + "projection.bias"});
        if (!m || !pw || !pb) return -1;
        const Act x = a;
        ++launches;
        b2sd_launch_record r{};
        r.kind = B2SD_LAUNCH_HED_PROJECT;
        r.hed_project = b2sd_hed_project_args{x.p, x.ld, x.c, (int64_t)x.h * x.w, pw, pb, m};
        prog_frame.push_back(Op([x, pw, pb, m](cudaStream_t st) { return hed_project_launch(x.p, x.ld, x.c, (long)x.h * x.w, pw, pb, m, st); },
                                "hed_project " + p, r));
        f.maps[b] = m; f.hs[b] = a.h; f.ws[b] = a.w;
    }
    f.levels = 5; f.h = H; f.w = W;
    f.out = static_cast<uint8_t*>(prog.alloc((size_t)H * W * 3));
    Act edge = new_act(1, H, W, 1);
    if (!f.out || !edge.p) return -1;
    f.edge_f16 = edge.p;
    ++launches;
    b2sd_launch_record r{};
    r.kind = B2SD_LAUNCH_HED_FUSE;
    for (int k = 0; k < 5; ++k) { r.hed_fuse.maps[k] = f.maps[k]; r.hed_fuse.hs[k] = f.hs[k]; r.hed_fuse.ws[k] = f.ws[k]; }
    r.hed_fuse.levels = f.levels; r.hed_fuse.h = f.h; r.hed_fuse.w = f.w; r.hed_fuse.out = f.out; r.hed_fuse.edge_f16 = f.edge_f16;
    prog_frame.push_back(Op([f](cudaStream_t st) { return hed_fuse_launch(f, st); }, "hed_fuse", r));
    taps["control"] = edge;
    *control = f.out;
    return 0;
}

b2sd_launch_record canny_ccl_record(const CannyCclArgs& a, int stage) {
    b2sd_launch_record r{};
    r.kind = B2SD_LAUNCH_CANNY_CCL;
    r.canny_ccl = b2sd_canny_ccl_args{a.cls, a.parent, a.flag, a.out, a.h, a.w, stage};
    return r;
}

// controlnet_aux's CannyDetector (cv2.Canny, aperture 3, L1 gradient) at the engine's resolution: canny_head (launched by the
// step, outside the graph) classifies every pixel of the frame; here the four hysteresis launches turn the class map into
// the u8 edge image (3 channels).  A fixed launch count, no grid-wide barrier: each launch waits for the previous one.
int b2sd_engine::build_canny(const uint8_t** control, cudaStream_t) {
    const int H = cfg.height, W = cfg.width;
    canny = CannyCclArgs{};
    canny.h = H; canny.w = W;
    canny.cls = canny_cls = static_cast<uint8_t*>(prog.alloc((size_t)H * W));
    canny.parent = static_cast<int*>(prog.alloc((size_t)H * W * sizeof(int)));
    canny.flag = static_cast<uint8_t*>(prog.alloc((size_t)H * W));
    canny.out = static_cast<uint8_t*>(prog.alloc((size_t)H * W * 3));
    if (!canny.cls || !canny.parent || !canny.flag || !canny.out) {
        b2_set_error("canny: buffer allocation failed");
        return -1;
    }
    ++launches;   // canny_head
    static const char* label[CANNY_CCL_STAGES] = {"canny_ccl local", "canny_ccl merge", "canny_ccl flag", "canny_ccl out"};
    for (int st = 0; st < CANNY_CCL_STAGES; ++st) {
        const CannyCclArgs a = canny;
        ++launches;
        prog_frame.push_back(Op([a, st](cudaStream_t q) { return canny_ccl_launch(a, st, q); }, label[st], canny_ccl_record(a, st)));
    }
    u8_taps["canny_class"] = U8Tap{canny.cls, H, W, 1};
    u8_taps["canny"] = U8Tap{canny.out, H, W, 3};
    *control = canny.out;
    return 0;
}

// ControlNetModel body: conv_in(x) + cond (broadcast to every stream-batch slot), the UNet's down blocks and mid block under the
// "controlnet." prefix with its own time embedding, then the zero convs: skips[k] <- skips[k] + controlnet_down_blocks.k(f_k),
// *mid <- *mid + controlnet_mid_block(f_mid), each one 1x1 contraction with the UNet tensor as its epilogue residual, written
// to a new buffer.  Each slot's residual is scaled by its conditioning scale (cn_scale, read when the launch runs: diffusers
// multiplies the zero conv's output, bias included, by controlnet_conditioning_scale).  Net i > 0 reads its own prefix, time
// embedding and row of scales, and its zero convs take the previous net's outputs as their residuals: the nets' residuals
// are summed into the skips as ((skip + r_0) + r_1) + ...
int b2sd_engine::build_controlnet(int net, const Act& cond, std::vector<Act>& skips, Act* mid, cudaStream_t s) {
    const std::string P = cn_prefix(net);
    const std::string tap = net == 0 ? "cn" : "cn" + std::to_string(net);
    const int B = cfg.batch, nlev = 4;
    const int* ch = cfg.block_out_channels;
    float* cn_temb = this->cn_temb[net];
    cur = P + "conv_in";
    allow_swap = true;
    Act h = new_act(B, lh, lw, ch[0]);
    {
        SmallConvArgs a{};
        a.wt = small_w(P + "conv_in.weight", s);
        a.bias = vec({P + "conv_in.bias"});
        if (!a.wt || !a.bias || !h.p) return -1;
        a.x = x_in.p; a.y = h.p; a.ldy = h.ld; a.nb = B; a.h = lh; a.w_ = lw; a.cin = 4; a.cout = ch[0]; a.in_h = lh; a.in_w = lw;
        a.res = cond.p; a.ldr = cond.ld; a.res_bstride = 0;
        ++launches;
        prog_frame.push_back(Op([a](cudaStream_t st) { return smallconv_launch(a, st); }, "smallconv " + P + "conv_in", smallconv_record(a)));
    }
    taps[tap + ".conv_in"] = h;
    std::vector<Act> feats{h};
    for (int i = 0; i < nlev; ++i) {
        const std::string bp = P + "down_blocks." + std::to_string(i);
        for (int j = 0; j < cfg.layers_per_block; ++j) {
            Act o;
            TRY(build_resnet(bp + ".resnets." + std::to_string(j) + ".", h, nullptr, ch[i], cn_temb, &o, s));
            h = o;
            if (cfg.down_attn[i]) {
                TRY(build_transformer(bp + ".attentions." + std::to_string(j) + ".", h, cfg.heads[i], &o, s));
                h = o;
            }
            feats.push_back(h);
        }
        if (i != nlev - 1) {
            Act o = new_act(B, h.h / 2, h.w / 2, ch[i]);
            const std::string k = bp + ".downsamplers.0.conv.";
            TRY(add_conv(prog_frame, h, k + "weight", k + "bias", 9, 2, o, 0, nullptr, s));
            h = o;
            feats.push_back(h);
        }
    }
    {
        Act o;
        TRY(build_resnet(P + "mid_block.resnets.0.", h, nullptr, ch[nlev - 1], cn_temb, &o, s)); h = o;
        TRY(build_transformer(P + "mid_block.attentions.0.", h, cfg.heads[nlev - 1], &o, s)); h = o;
        TRY(build_resnet(P + "mid_block.resnets.1.", h, nullptr, ch[nlev - 1], cn_temb, &o, s)); h = o;
    }
    if (feats.size() != skips.size()) {
        b2_set_error("controlnet: %zu down residuals for %zu UNet skips", feats.size(), skips.size());
        return -1;
    }
    allow_swap = false;
    if (net == 0) {   // every net's row of scales, [nets][B]  (`cond` is the embedding here)
        cn_scale = static_cast<float*>(this->cond[COND_TIME].take((size_t)cfg.controlnet * B * sizeof(float)));
        if (!cn_scale) return -1;
    }
    float* scale = cn_scale + (size_t)net * B;
    auto tap_both = [&](const std::string& name, const Act& a) {   // net 0 also keeps its single-net names
        taps[tap + name] = a;
        if (net == 0) taps["cn0" + name] = a;
    };
    for (size_t k = 0; k < feats.size(); ++k) {
        const std::string w = P + "controlnet_down_blocks." + std::to_string(k);
        Act o = new_act(skips[k].n, skips[k].h, skips[k].w, skips[k].c);
        TRY(add_conv(prog_frame, feats[k], w + ".weight", w + ".bias", 1, 1, o, 0, &skips[k], s, 1.f, 1.f, scale));
        skips[k] = o;
        tap_both(".res." + std::to_string(k), o);
    }
    Act o = new_act(mid->n, mid->h, mid->w, mid->c);
    TRY(add_conv(prog_frame, h, P + "controlnet_mid_block.weight", P + "controlnet_mid_block.bias", 1, 1, o, 0, mid, s, 1.f, 1.f,
                 scale));
    *mid = o;
    tap_both(".mid", o);
    allow_swap = true;
    return 0;
}

// ---- AutoencoderKL (diffusers autoencoder_kl.py / vae.py Encoder, Decoder; cfg.vae == B2SD_VAE_KL) -------------------------------
// A parameter as fp32 on the host (exact weight foldings at build time; read before the pack-only raw copies are released).
std::vector<float> b2sd_engine::host_copy(const std::string& key) {
    const Raw* r = get(key);
    if (!r || !r->p) {
        if (r) b2_set_error("parameter '%s' was released before the weight folding that needs it", key.c_str());
        return {};
    }
    std::vector<__half> h((size_t)r->numel());
    if (cudaMemcpy(h.data(), r->p, h.size() * 2, cudaMemcpyDeviceToHost) != cudaSuccess) {
        b2_set_error("host copy of '%s' failed", key.c_str());
        return {};
    }
    std::vector<float> f(h.size());
    for (size_t i = 0; i < h.size(); ++i) f[i] = __half2float(h[i]);
    return f;
}

// A parameter the engine computes from loaded ones, stored like a loaded parameter (fp16; packed / exported like the others).
int b2sd_engine::derive(const std::string& name, const std::vector<int64_t>& shape, const std::vector<float>& v) {
    Raw r;
    r.shape = shape;
    r.derived = true;
    r.pack_only = shape.size() == 4 && shape[2] == 3;
    if ((size_t)r.numel() != v.size()) {
        b2_set_error("derived parameter '%s': %zu values for %ld elements", name.c_str(), v.size(), r.numel());
        return -1;
    }
    std::vector<__half> h(v.size());
    for (size_t i = 0; i < v.size(); ++i) h[i] = __float2half_rn(v[i]);
    r.p = static_cast<__half*>((r.pack_only ? raw_only : weights).alloc(h.size() * 2));
    if (!r.p || cudaMemcpy(r.p, h.data(), h.size() * 2, cudaMemcpyHostToDevice) != cudaSuccess) {
        b2_set_error("derived parameter '%s': upload failed", name.c_str());
        return -1;
    }
    if (shape.size() == 1)
        for (auto x : h) r.host.push_back(__half2float(x));
    raw[name] = std::move(r);
    return 0;
}

// fp32 device constant vector (cached with the other fp32 vectors)
const float* b2sd_engine::const_vec(const std::string& name, const std::vector<float>& v) {
    auto it = fvec.find(name);
    if (it != fvec.end()) return it->second;
    float* d = static_cast<float*>(weights.alloc(v.size() * sizeof(float)));
    if (!d || cudaMemcpy(d, v.data(), v.size() * sizeof(float), cudaMemcpyHostToDevice) != cudaSuccess) return nullptr;
    fvec[name] = d;
    fvec_bytes[name] = v.size() * sizeof(float);
    return d;
}

// Mid-block Attention(heads=1, dim_head=C, residual_connection=True, bias=True, upcast_softmax=True): GroupNorm (eps 1e-6, no
// SiLU) -> one [q | k | v] GEMM with bias, V stored transposed -> single-head attention (attn_d512_kernel) -> to_out.0 + x.
int b2sd_engine::build_vae_attention(const std::string& p, const Act& x, Act* out, cudaStream_t s) {
    cur = p;
    allow_swap = false;
    const int C = x.c, M = x.n * x.h * x.w;
    if (x.n != 1 || C != 512) {
        b2_set_error("vae attention %s: single image with 512 channels expected (got %d x %d)", p.c_str(), x.n, C);
        return -1;
    }
    Act n = new_act(1, x.h, x.w, C);
    TRY(add_groupnorm(x, nullptr, p + "group_norm", n, 1e-6f, 0));
    std::vector<int> id(C);
    for (int i = 0; i < C; ++i) id[i] = i;
    __half* w = pack_rows(p + "qkv", {{p + "to_q.weight", id}, {p + "to_k.weight", id}, {p + "to_v.weight", id}}, C, s);
    if (!w) return -1;
    const float* bias = fvec.count(p + "qkv.bias") ? fvec[p + "qkv.bias"] : nullptr;
    if (!bias) {
        std::vector<float> b;
        for (const char* t : {"to_q.bias", "to_k.bias", "to_v.bias"}) {
            const Raw* r = get(p + t);
            if (!r) return -1;
            b.insert(b.end(), r->host.begin(), r->host.end());
        }
        bias = const_vec(p + "qkv.bias", b);
        if (!bias) return -1;
    }
    Act qk = new_act(1, 1, M, 2 * C);
    const long vt_ld = (M + 7) / 8 * 8;
    __half* vt = static_cast<__half*>(prog.alloc((size_t)C * vt_ld * 2));
    if (!vt || !qk.p) return -1;
    cudaMemsetAsync(vt, 0, (size_t)C * vt_ld * 2, s);   // pad columns must stay finite
    LinExtra ex; ex.out2 = vt; ex.ld2 = (int)vt_ld; ex.col2 = 2 * C;
    TRY(add_linear(prog_frame, tokens(n), w, 3 * C, C, bias, qk.p, 2 * C, nullptr, 0, 0, -1, &ex));
    Act ao = new_act(1, x.h, x.w, C);
    AttnDesc a{};
    a.q = qk.p; a.ldq = 2 * C;
    a.k = qk.p + C; a.ldk = 2 * C; a.k_bstride = 0; a.k_rows = M;
    a.vt = vt; a.ldvt = (int)vt_ld; a.vt_bstride = 0; a.vt_cols = M;
    a.out = ao.p; a.ldo = C;
    a.nb = 1; a.heads = 1; a.sq = M; a.skv = M; a.d_real = C; a.dp = C;
    AttnPlan plan;
    TRY(attn_plan(a, &plan));
    push_attn(plan, "attn " + p);
    const Raw* wo = get(p + "to_out.0.weight");
    if (!wo) return -1;
    *out = new_act(1, x.h, x.w, C);
    return add_linear(prog_frame, tokens(ao), wo->p, C, C, vec({p + "to_out.0.bias"}), out->p, C, x.p, x.ld);
}

// Encoder: conv_in (reads the caller's frame: `head`), 4 DownEncoderBlock2D (2 resnets, Downsample2D(padding=0) after levels
// 0-2), mid block, GroupNorm + SiLU.  Returns that last activation and the key of the latent conv that follows it:
// conv_out composed with rows 0-3 of quant_conv (the distribution's mean), an exact folding (a 1x1 conv after a conv).
// The image normalisation 2x - 1 = (2/255)(u8 - 127.5) is the smallconv offset input mode with 2/255 folded into the
// weights: zero padding then applies to 2x - 1, as in the model (a folded bias would be wrong on the border pixels).
int b2sd_engine::build_kl_encoder(Act* out, std::string* latent_conv, cudaStream_t s) {
    const std::string P = "vae.encoder.";
    const int H = cfg.height, W = cfg.width;
    allow_swap = false;
    cur = P + "conv_in";
    const std::string win = P + "conv_in.weight*2/255";
    if (!has(win)) {
        const Raw* r = get(P + "conv_in.weight");
        if (!r) return -1;
        std::vector<float> v = host_copy(P + "conv_in.weight");
        if (v.empty()) return -1;
        for (auto& x : v) x *= 2.0f / 255.0f;
        TRY(derive(win, r->shape, v));
    }
    const Raw* rin = get(win);
    if (!rin) return -1;
    const int c0 = (int)rin->shape[0];
    Act e = new_act(1, H, W, c0);
    head = SmallConvArgs{};
    head.wt = small_w(win, s);
    head.bias = vec({P + "conv_in.bias"});
    head.in_off = const_vec("vae:in_off", {127.5f, 127.5f, 127.5f});
    if (!head.wt || !head.bias || !head.in_off || !e.p) return -1;
    head.y = e.p; head.ldy = e.ld; head.nb = 1; head.h = H; head.w_ = W; head.cin = 3; head.cout = c0;
    head.flags = SC_IN_U8 | SC_IN_OFFSET;
    ++launches;
    for (int i = 0; i < 4; ++i) {
        const std::string bp = P + "down_blocks." + std::to_string(i);
        for (int j = 0; j < 2; ++j) {
            const Raw* w1 = get(bp + ".resnets." + std::to_string(j) + ".conv1.weight");
            if (!w1) return -1;
            Act o;
            TRY(build_resnet(bp + ".resnets." + std::to_string(j) + ".", e, nullptr, (int)w1->shape[0], nullptr, &o, s, 1e-6f));
            e = o;
        }
        if (i < 3) {
            Act o = new_act(1, e.h / 2, e.w / 2, e.c);
            TRY(add_conv(prog_frame, e, bp + ".downsamplers.0.conv.weight", bp + ".downsamplers.0.conv.bias", 9, 2, o, IG_PAD0,
                         nullptr, s));
            e = o;
        }
        taps["vae.enc.down." + std::to_string(i)] = e;
    }
    {
        Act o;
        TRY(build_resnet(P + "mid_block.resnets.0.", e, nullptr, e.c, nullptr, &o, s, 1e-6f)); e = o;
        TRY(build_vae_attention(P + "mid_block.attentions.0.", e, &o, s)); e = o;
        TRY(build_resnet(P + "mid_block.resnets.1.", e, nullptr, e.c, nullptr, &o, s, 1e-6f)); e = o;
        taps["vae.enc.mid"] = e;
    }
    *out = new_act(1, e.h, e.w, e.c);
    TRY(add_groupnorm(e, nullptr, P + "conv_norm_out", *out, 1e-6f, 1));
    *latent_conv = P + "conv_out+quant_conv";
    if (!has(*latent_conv + ".weight")) {
        const Raw* wc = get(P + "conv_out.weight");
        const Raw* wq = get("vae.quant_conv.weight");
        if (!wc || !wq) return -1;
        const int co = (int)wc->shape[0], ci = (int)wc->shape[1];
        if (co != 8 || wq->numel() != 64) {
            b2_set_error("vae: conv_out has %d channels and quant_conv %ld weights (8 and 8x8 expected)", co, wq->numel());
            return -1;
        }
        std::vector<float> w = host_copy(P + "conv_out.weight"), b = host_copy(P + "conv_out.bias"), q = host_copy("vae.quant_conv.weight"),
                           qb = host_copy("vae.quant_conv.bias");
        if (w.empty() || b.empty() || q.empty() || qb.empty()) return -1;
        const size_t per = (size_t)ci * 9;
        std::vector<float> wf(4 * per, 0.f), bf(4, 0.f);
        for (int o = 0; o < 4; ++o) {
            double bo = qb[o];
            for (int j = 0; j < 8; ++j) {
                const float qv = q[o * 8 + j];
                for (size_t k = 0; k < per; ++k) wf[o * per + k] += qv * w[j * per + k];
                bo += (double)qv * b[j];
            }
            bf[o] = (float)bo;
        }
        TRY(derive(*latent_conv + ".weight", {4, ci, 3, 3}, wf));
        TRY(derive(*latent_conv + ".bias", {4}, bf));
    }
    return 0;
}

// Decoder on x0: post_quant_conv and 1/scaling_factor folded into conv_in's weights (exact: 1x1 before a conv).  post_quant_conv's
// bias is NOT folded into conv_in's bias -- conv_in zero-pads post_quant_conv's output, so its contribution differs on the
// border: it is computed once per program as conv_in(constant bias image) + conv_in.bias (same kernel, same zero padding) and
// added as the residual of the frame's conv_in.  Then the mid block, 4 UpDecoderBlock2D (3 resnets, nearest 2x + conv after
// levels 0-2), GroupNorm + SiLU, conv_out.  `image` holds the decoded image on the [0, 1] scale, (y + 1) / 2 (conv_out's epilogue:
// 0.5 * (acc + bias + 1)), which is what the TAESD decoder's last conv produces: the tails (post_u8 / post_f16) are shared.
int b2sd_engine::build_kl_decoder(const Act& x0, cudaStream_t s) {
    const std::string P = "vae.decoder.";
    allow_swap = false;
    cur = P + "conv_in";
    const float sf = cfg.vae_scaling_factor > 0.f ? cfg.vae_scaling_factor : 0.18215f;
    const std::string wkey = P + "conv_in+post_quant_conv.weight";
    if (!has(wkey)) {
        const Raw* wc = get(P + "conv_in.weight");
        const Raw* wq = get("vae.post_quant_conv.weight");
        if (!wc || !wq) return -1;
        const int co = (int)wc->shape[0];
        if (wc->shape[1] != 4 || wq->numel() != 16) {
            b2_set_error("vae: decoder conv_in takes %ld channels and post_quant_conv has %ld weights (4 and 4x4 expected)",
                         (long)wc->shape[1], wq->numel());
            return -1;
        }
        std::vector<float> w = host_copy(P + "conv_in.weight"), q = host_copy("vae.post_quant_conv.weight");
        if (w.empty() || q.empty()) return -1;
        std::vector<float> wf((size_t)co * 4 * 9, 0.f);
        for (int o = 0; o < co; ++o)
            for (int j = 0; j < 4; ++j)
                for (int t = 0; t < 9; ++t) {
                    double acc = 0.0;
                    for (int i = 0; i < 4; ++i) acc += (double)w[((size_t)o * 4 + i) * 9 + t] * q[i * 4 + j];
                    wf[((size_t)o * 4 + j) * 9 + t] = (float)(acc / sf);
                }
        TRY(derive(wkey, {co, 4, 3, 3}, wf));
    }
    const Raw* rw = get(wkey);
    const Raw* pqb = get("vae.post_quant_conv.bias");
    if (!rw || !pqb || pqb->host.size() != 4) {
        if (rw && pqb) b2_set_error("vae: post_quant_conv.bias must have 4 elements");
        return -1;
    }
    const int cm = (int)rw->shape[0];
    Act bmap = new_act(1, lh, lw, cm), cst = new_act(1, lh, lw, 4), h = new_act(1, lh, lw, cm);
    if (!bmap.p || !cst.p || !h.p) return -1;
    {
        std::vector<__half> c((size_t)lh * lw * 4);
        for (size_t i = 0; i < c.size(); ++i) c[i] = __float2half_rn(pqb->host[i % 4]);
        CUDA_OK(cudaMemcpyAsync(cst.p, c.data(), c.size() * 2, cudaMemcpyHostToDevice, s));
        SmallConvArgs m{};
        m.x = cst.p; m.wt = small_w(P + "conv_in.weight", s); m.bias = vec({P + "conv_in.bias"});
        if (!m.wt || !m.bias) return -1;
        m.y = bmap.p; m.ldy = cm; m.nb = 1; m.h = lh; m.w_ = lw; m.cin = 4; m.cout = cm; m.in_h = lh; m.in_w = lw;
        TRY(smallconv_launch(m, s));
        CUDA_OK(cudaStreamSynchronize(s));   // the host constant image dies with this scope
    }
    {
        SmallConvArgs a{};
        a.x = x0.p; a.wt = small_w(wkey, s); a.bias = nullptr;
        if (!a.wt) return -1;
        a.y = h.p; a.ldy = h.ld; a.nb = 1; a.h = lh; a.w_ = lw; a.cin = 4; a.cout = cm; a.in_h = lh; a.in_w = lw;
        a.res = bmap.p; a.ldr = bmap.ld; a.res_bstride = 0;
        ++launches;
        prog_frame.push_back(Op([a](cudaStream_t st) { return smallconv_launch(a, st); }, "smallconv vae.decoder.conv_in", smallconv_record(a)));
    }
    {
        Act o;
        TRY(build_resnet(P + "mid_block.resnets.0.", h, nullptr, h.c, nullptr, &o, s, 1e-6f)); h = o;
        TRY(build_vae_attention(P + "mid_block.attentions.0.", h, &o, s)); h = o;
        TRY(build_resnet(P + "mid_block.resnets.1.", h, nullptr, h.c, nullptr, &o, s, 1e-6f)); h = o;
        taps["vae.dec.mid"] = h;
    }
    for (int i = 0; i < 4; ++i) {
        const std::string bp = P + "up_blocks." + std::to_string(i);
        for (int j = 0; j < 3; ++j) {
            const Raw* w1 = get(bp + ".resnets." + std::to_string(j) + ".conv1.weight");
            if (!w1) return -1;
            Act o;
            TRY(build_resnet(bp + ".resnets." + std::to_string(j) + ".", h, nullptr, (int)w1->shape[0], nullptr, &o, s, 1e-6f));
            h = o;
        }
        if (i < 3) {
            Act up = new_act(1, h.h * 2, h.w * 2, h.c);
            const Act hin = h;
            ++launches;
            prog_frame.push_back(Op([hin, up](cudaStream_t st) { return upsample2x_launch(hin.p, up.p, hin.n, hin.h, hin.w, hin.c, st); }, "upsample2x",
                                    upsample2x_record(hin.p, up.p, hin.n, hin.h, hin.w, hin.c)));
            Act o = new_act(1, up.h, up.w, h.c);
            TRY(add_conv(prog_frame, up, bp + ".upsamplers.0.conv.weight", bp + ".upsamplers.0.conv.bias", 9, 1, o, 0, nullptr, s));
            h = o;
        }
        taps["vae.dec.up." + std::to_string(i)] = h;
    }
    Act nout = new_act(1, h.h, h.w, h.c);
    TRY(add_groupnorm(h, nullptr, P + "conv_norm_out", nout, 1e-6f, 1));
    const std::string bkey = P + "conv_out.bias+1";
    if (!has(bkey)) {
        const Raw* b = get(P + "conv_out.bias");
        if (!b) return -1;
        std::vector<float> v(b->host);
        for (auto& x : v) x += 1.f;
        TRY(derive(bkey, b->shape, v));
    }
    image = new_act(1, cfg.height, cfg.width, 3, 8);
    return add_conv(prog_frame, nout, P + "conv_out.weight", bkey, 9, 1, image, 0, nullptr, s, 0.5f);
}

int b2sd_engine::build_program(cudaStream_t s) {
    prog.reset();
    prog_frame.clear(); prog_prompt.clear(); prog_time.clear(); prog_image.clear();
    taps.clear();
    u8_taps.clear();
    launches = 0;
    drop_graphs();
    const int B = cfg.batch, H = cfg.height, W = cfg.width;
    const int* ch = cfg.block_out_channels;
    const int nlev = 4;
    {
        // LayerNorm row statistics of every transformer block (3 per block, [tokens][2] 64-bit words), one slab that a single
        // memset node clears at the start of each frame
        long words = 0;
        for (int i = 0; i < nlev; ++i) {
            const long tokens_i = (long)B * (lh >> i) * (lw >> i);
            int blocks_i = (cfg.down_attn[i] ? cfg.layers_per_block + (cfg.layers_per_block + 1) : 0) + (i == nlev - 1 ? 1 : 0);
            blocks_i += cfg.controlnet * ((cfg.down_attn[i] ? cfg.layers_per_block : 0) + (i == nlev - 1 ? 1 : 0));
            words += 3 * 2 * tokens_i * blocks_i;
        }
        ln_stats_cap = (size_t)words;
        ln_stats_used = 0;
        ln_stats = static_cast<unsigned long long*>(prog.alloc(ln_stats_cap * sizeof(unsigned long long)));
        if (!ln_stats) return -1;
    }
    {
        // the conditioning blocks, sized from the shapes build_transformer (K [L][Cp], V^T [Cp][Lpad] per block) and build_resnet
        // (time bias [B][cout] per resnet) take from them, and zeroed once (V^T's pad columns are never written)
        const int L = cfg.ctx_tokens, Lpad = 128 * ((L + 127) / 128), lpb = cfg.layers_per_block, cn = cfg.controlnet;
        auto r = [](size_t b) { return (b + 1023) & ~size_t(1023); };
        size_t bytes[2] = {0, 0};
        for (int i = 0; i < nlev; ++i) {
            const int d_real = ch[i] / cfg.heads[i], dp = d_real <= 64 ? 64 : (d_real <= 128 ? 128 : 192);
            const size_t Cp = (size_t)cfg.heads[i] * dp;
            // UNet down + up blocks (and the ControlNet's down blocks) of this level, the mid blocks at the last one
            int transformers = cfg.down_attn[i] ? lpb + (lpb + 1) + cn * lpb : 0;
            int resnets = lpb + (lpb + 1) + cn * lpb;
            if (i == nlev - 1) {
                transformers += 1 + cn;
                resnets += 2 * (1 + cn);
            }
            bytes[COND_PROMPT] += transformers * (r(L * Cp * 2) + r(Cp * Lpad * 2));
            if (cfg.ip_tokens)   // the UNet's own (not the ControlNet's): image K [64][Cp] and V^T [Cp][64]
                bytes[COND_PROMPT] += (transformers - cn * (cfg.down_attn[i] ? lpb : 0) - (i == nlev - 1 ? cn : 0)) *
                                      2 * r((size_t)ATTN_IP_KEYS * Cp * 2);
            bytes[COND_TIME] += resnets * r((size_t)B * ch[i] * sizeof(float));
        }
        if (cfg.controlnet) bytes[COND_TIME] += r((size_t)cfg.controlnet * B * sizeof(float));   // the per-slot ControlNet scales
        if (cfg.ip_tokens) bytes[COND_PROMPT] += r(sizeof(int));   // ip_count
        for (int k = 0; k < 2; ++k) {
            CondBlock& b = cond[k];
            b.cap = bytes[k];
            b.used = 0;
            b.held = COND_UNKNOWN;
            b.p = static_cast<char*>(prog.alloc(b.cap));
            b.global = static_cast<char*>(prog.alloc(b.cap));
            if (!b.p || !b.global) return -1;
            CUDA_OK(cudaMemsetAsync(b.p, 0, b.cap, s));
            CUDA_OK(cudaMemsetAsync(b.global, 0, b.cap, s));
        }
        ip_count = cfg.ip_tokens ? static_cast<int*>(cond[COND_PROMPT].take(sizeof(int))) : nullptr;
    }

    allow_swap = false;
    const bool kl = cfg.vae == B2SD_VAE_KL;
    Act e;
    std::string latent_conv;   // the encoder's last conv (its epilogue adds the noise)
    int li = 1;
    if (kl) {
        TRY(build_kl_encoder(&e, &latent_conv, s));
    } else {
    // ================= TAESD encoder (EncoderTiny) =================
    e = new_act(1, H, W, 64);
    {
        head = SmallConvArgs{};
        head.wt = small_w("vae.encoder.layers.0.weight", s);
        if (!head.wt) return -1;
        head.bias = vec({"vae.encoder.layers.0.bias"});
        head.y = e.p; head.ldy = e.ld; head.nb = 1; head.h = H; head.w_ = W; head.cin = 3; head.cout = 64;
        head.flags = SC_IN_U8;
        if (!head.bias) return -1;
        ++launches;
    }
    const int enc_blocks[4] = {1, 3, 3, 3};
    for (int st = 0; st < 4; ++st) {
        if (st > 0) {
            Act dwn = new_act(1, e.h / 2, e.w / 2, 64);
            TRY(add_conv(prog_frame, e, "vae.encoder.layers." + std::to_string(li) + ".weight", "", 9, 2, dwn, 0, nullptr, s));
            e = dwn;
            ++li;
        }
        for (int k = 0; k < enc_blocks[st]; ++k) {
            Act o;
            TRY(build_taesd_block("vae.encoder.layers." + std::to_string(li), e, &o, s));
            e = o;
            ++li;
        }
    }
    latent_conv = "vae.encoder.layers." + std::to_string(li);
    }
    // each ControlNet's conditioning embedding of this frame's control image: batch 1, latent resolution, C0 channels
    Act cond[B2SD_MAX_CONTROLNETS];
    const uint8_t* shared_control[3] = {};   // per processor: HED's / Canny's edge map, once a net reads it
    for (int i = 0; i < cfg.controlnet; ++i) TRY(build_cond_embedding(i, shared_control, &cond[i], s));
    {
        // latent head + StreamDiffusion.encode_image add-noise: x_t = alpha0 * z + beta0 * init_noise[0]
        // (AutoencoderKL: z = scaling_factor * mean, the scale applied with alpha0 in the epilogue)
        Act xt;  // slot 0 of the UNet input batch
        xt.p = x_in.p; xt.n = 1; xt.h = lh; xt.w = lw; xt.c = 4; xt.ld = 4;
        Act nz = xt;
        nz.p = noise;
        const float zscale = kl ? (cfg.vae_scaling_factor > 0.f ? cfg.vae_scaling_factor : 0.18215f) : 1.f;
        idx_enc_end = prog_frame.size();   // everything before this conv only touches this engine's own activations
        TRY(add_conv(prog_frame, e, latent_conv + ".weight", latent_conv + ".bias", 9, 1, xt, 0, &nz, s, coef_host[0][0] * zscale,
                     coef_host[1][0]));
        taps["x_t"] = xt;
    }
    taps["unet_in"] = x_in;

    allow_swap = true;
    // ================= UNet2DConditionModel =================
    Act h = new_act(B, lh, lw, ch[0]);
    {
        SmallConvArgs a{};
        a.wt = small_w("conv_in.weight", s);
        if (!a.wt) return -1;
        a.x = x_in.p; a.bias = vec({"conv_in.bias"});
        a.y = h.p; a.ldy = h.ld; a.nb = B; a.h = lh; a.w_ = lw; a.cin = 4; a.cout = ch[0]; a.in_h = lh; a.in_w = lw;
        if (!a.bias) return -1;
        ++launches;
        prog_frame.push_back(Op([a](cudaStream_t st) { return smallconv_launch(a, st); }, "smallconv", smallconv_record(a)));
    }
    taps["conv_in"] = h;
    std::vector<Act> skips{h};
    for (int i = 0; i < nlev; ++i) {
        for (int j = 0; j < cfg.layers_per_block; ++j) {
            Act o;
            const std::string bp = "down_blocks." + std::to_string(i);
            TRY(build_resnet(bp + ".resnets." + std::to_string(j) + ".", h, nullptr, ch[i], temb, &o, s));
            h = o;
            if (cfg.down_attn[i]) {
                TRY(build_transformer(bp + ".attentions." + std::to_string(j) + ".", h, cfg.heads[i], &o, s));
                h = o;
            }
            skips.push_back(h);
            taps["down." + std::to_string(i) + "." + std::to_string(j)] = h;
        }
        if (i != nlev - 1) {
            Act o = new_act(B, h.h / 2, h.w / 2, ch[i]);
            const std::string k = "down_blocks." + std::to_string(i) + ".downsamplers.0.conv.";
            TRY(add_conv(prog_frame, h, k + "weight", k + "bias", 9, 2, o, 0, nullptr, s));
            h = o;
            skips.push_back(h);
        }
    }
    {
        Act o;
        TRY(build_resnet("mid_block.resnets.0.", h, nullptr, ch[nlev - 1], temb, &o, s)); h = o;
        TRY(build_transformer("mid_block.attentions.0.", h, cfg.heads[nlev - 1], &o, s)); h = o;
        TRY(build_resnet("mid_block.resnets.1.", h, nullptr, ch[nlev - 1], temb, &o, s)); h = o;
        taps["mid"] = h;
    }
    // ControlNet: its down path + mid block over the same x / timesteps / prompt; the zero convs add its 12 + 1 residuals to the
    // skips the up path concatenates and to the mid-block output (the UNet's own down path above used them unmodified)
    for (int i = 0; i < cfg.controlnet; ++i) TRY(build_controlnet(i, cond[i], skips, &h, s));
    for (int i = 0; i < nlev; ++i) {
        const int co = ch[nlev - 1 - i];
        const int hd = cfg.heads[nlev - 1 - i];
        const bool attn = cfg.down_attn[nlev - 1 - i] != 0;
        for (int j = 0; j < cfg.layers_per_block + 1; ++j) {
            Act sk = skips.back();
            skips.pop_back();
            Act o;
            const std::string bp = "up_blocks." + std::to_string(i);
            TRY(build_resnet(bp + ".resnets." + std::to_string(j) + ".", h, &sk, co, temb, &o, s));
            h = o;
            if (attn) {
                TRY(build_transformer(bp + ".attentions." + std::to_string(j) + ".", h, hd, &o, s));
                h = o;
            }
            taps["up." + std::to_string(i) + "." + std::to_string(j)] = h;
        }
        if (i != nlev - 1) {
            Act up = new_act(B, h.h * 2, h.w * 2, co);
            const Act hin = h;
            ++launches;
            prog_frame.push_back(Op([hin, up](cudaStream_t st) { return upsample2x_launch(hin.p, up.p, hin.n, hin.h, hin.w, hin.c, st); }, "upsample2x",
                                    upsample2x_record(hin.p, up.p, hin.n, hin.h, hin.w, hin.c)));
            Act o = new_act(B, up.h, up.w, co);
            const std::string k = "up_blocks." + std::to_string(i) + ".upsamplers.0.conv.";
            TRY(add_conv(prog_frame, up, k + "weight", k + "bias", 9, 1, o, 0, nullptr, s));
            h = o;
        }
    }
    Act nout = new_act(B, lh, lw, ch[0]);
    TRY(add_groupnorm(h, nullptr, "conv_norm_out", nout, 1e-5f, 1));
    Act eps = new_act(B, lh, lw, 4);
    TRY(add_conv(prog_frame, nout, "conv_out.weight", "conv_out.bias", 9, 1, eps, 0, nullptr, s));
    taps["eps"] = eps;
    // ================= scheduler_step_batch + stream-batch buffer update =================
    Act x0 = new_act(1, lh, lw, 4);
    {
        __half* xp = x_in.p; const __half* ep = eps.p; const __half* np_ = noise; const float* cf = coef; __half* op = x0.p;
        const int T = B, hw = lh * lw, dan = cfg.do_add_noise;
        ++launches;
        b2sd_launch_record r{};
        r.kind = B2SD_LAUNCH_LCM_STEP;
        r.lcm_step = b2sd_lcm_step_args{xp, ep, np_, cf, op, T, hw, dan};
        prog_frame.push_back(Op([=](cudaStream_t st) { return lcm_step_launch(xp, ep, np_, cf, op, T, hw, dan, st); }, "lcm_step", r));
        idx_unet_end = prog_frame.size();
    }
    taps["x0"] = x0;
    allow_swap = false;
    if (kl) {
        TRY(build_kl_decoder(x0, s));
    } else {
    // ================= TAESD decoder (DecoderTiny) =================
    Act dcur = new_act(1, lh, lw, 64);
    {
        SmallConvArgs a{};
        a.wt = small_w("vae.decoder.layers.0.weight", s);
        if (!a.wt) return -1;
        a.x = x0.p; a.bias = vec({"vae.decoder.layers.0.bias"});
        a.y = dcur.p; a.ldy = dcur.ld; a.nb = 1; a.h = lh; a.w_ = lw; a.cin = 4; a.cout = 64; a.in_h = lh; a.in_w = lw;
        a.flags = SC_IN_TANH3 | SC_OUT_RELU;
        if (!a.bias) return -1;
        ++launches;
        prog_frame.push_back(Op([a](cudaStream_t st) { return smallconv_launch(a, st); }, "smallconv", smallconv_record(a)));
    }
    li = 2;
    const int dec_blocks[4] = {3, 3, 3, 1};
    for (int st = 0; st < 4; ++st) {
        for (int k = 0; k < dec_blocks[st]; ++k) {
            Act o;
            TRY(build_taesd_block("vae.decoder.layers." + std::to_string(li), dcur, &o, s));
            dcur = o;
            ++li;
        }
        if (st != 3) {
            Act up = new_act(1, dcur.h * 2, dcur.w * 2, 64);
            const Act hin = dcur;
            ++launches;
            prog_frame.push_back(Op([hin, up](cudaStream_t s2) { return upsample2x_launch(hin.p, up.p, hin.n, hin.h, hin.w, hin.c, s2); }, "upsample2x",
                                    upsample2x_record(hin.p, up.p, hin.n, hin.h, hin.w, hin.c)));
            ++li;  // nn.Upsample
            Act o = new_act(1, up.h, up.w, 64);
            TRY(add_conv(prog_frame, up, "vae.decoder.layers." + std::to_string(li) + ".weight", "", 9, 1, o, 0, nullptr, s));
            dcur = o;
            ++li;
        } else {
            image = new_act(1, H, W, 3, 8);
            const std::string k = "vae.decoder.layers." + std::to_string(li);
            TRY(add_conv(prog_frame, dcur, k + ".weight", k + ".bias", 9, 1, image, 0, nullptr, s));
        }
    }
    }
    taps["image"] = image;
    ++launches;  // post_u8 tail
    if (ln_stats_used) {
        unsigned long long* sp = ln_stats;
        const size_t bytes = ln_stats_used * sizeof(unsigned long long);
        // first op of the UNet stage (the statistics belong to the transformer blocks)
        prog_frame.insert(prog_frame.begin() + idx_enc_end, Op([sp, bytes](cudaStream_t st) {
            if (cudaMemsetAsync(sp, 0, bytes, st) != cudaSuccess) { b2_set_error("memset of the LayerNorm statistics failed"); return -1; }
            return 0; }, "memset ln_stats"));
        idx_unet_end += 1;
    }
    CUDA_OK(cudaStreamSynchronize(s));
    built = true;
    return 0;
}

// ---- stream states -------------------------------------------------------------------------------
static size_t state_bytes(const b2sd_engine* h) { return (size_t)(h->cfg.batch - 1) * h->lh * h->lw * 4 * sizeof(__half); }

static int state_new(const b2sd_engine* h, cudaStream_t s, b2sd_state** out) {
    b2sd_state* st = new b2sd_state;
    st->family = h->ws->family;
    st->batch = h->cfg.batch; st->height = h->cfg.height; st->width = h->cfg.width;
    st->bytes = state_bytes(h);
    st->canny = h->reads_canny();
    cudaError_t e = cudaEventCreateWithFlags(&st->done, cudaEventDisableTiming);
    if (e == cudaSuccess && st->bytes) e = cudaMallocAsync(reinterpret_cast<void**>(&st->buf), st->bytes, s);
    if (e == cudaSuccess && st->bytes) e = cudaMemsetAsync(st->buf, 0, st->bytes, s);
    if (e == cudaSuccess) e = cudaEventRecord(st->done, s);
    if (e != cudaSuccess) {
        b2_set_error("b2sd_state_create: %s", cudaGetErrorString(e));
        if (st->buf) cudaFreeAsync(st->buf, s);
        if (st->done) cudaEventDestroy(st->done);
        delete st;
        return -1;
    }
    *out = st;
    return 0;
}

static int state_free(b2sd_state* st, cudaStream_t s) {
    cudaError_t e = cudaSuccess;
    if (st->buf) {
        e = cudaStreamWaitEvent(s, st->done, 0);
        if (e == cudaSuccess) e = cudaFreeAsync(st->buf, s);
    }
    cudaEventDestroy(st->done);   // a recorded, not yet completed event is released once the device reaches it
    delete st;
    if (e != cudaSuccess) {
        b2_set_error("b2sd_state_destroy: %s", cudaGetErrorString(e));
        return -1;
    }
    return 0;
}

static int state_reset(b2sd_state* st, cudaStream_t s) {
    CUDA_OK(cudaStreamWaitEvent(s, st->done, 0));
    if (st->bytes) CUDA_OK(cudaMemsetAsync(st->buf, 0, st->bytes, s));
    CUDA_OK(cudaEventRecord(st->done, s));
    return 0;
}

// ---- conditioning blocks ----------------------------------------------------------------------------
// The engine's global ControlNet scales into the time block, as a kernel argument: stream-ordered, and no host buffer has to
// outlive the call
struct Scales16 { float v[16]; };
__global__ void write_scales_kernel(float* dst, Scales16 v, int n) {
    if ((int)threadIdx.x < n) dst[threadIdx.x] = v.v[threadIdx.x];
}
static int write_global_scales(b2sd_engine* h, cudaStream_t s) {
    if (!h->cn_scale) return 0;
    for (int i = 0; i < h->cfg.controlnet; ++i) {   // one net's row per launch
        Scales16 v;
        memcpy(v.v, h->cn_scale_global[i], sizeof(v.v));
        write_scales_kernel<<<1, 32, 0, s>>>(h->cn_scale + (size_t)i * h->cfg.batch, v, h->cfg.batch);
        CUDA_OK(cudaGetLastError());
    }
    return 0;
}

// Block k now holds the lane's global values (after b2sd_prepare / b2sd_set_*, which computed them into it): keep a copy to rebind.
static int keep_global(b2sd_engine* h, int k, cudaStream_t s) {
    auto& b = h->cond[k];
    CUDA_OK(cudaMemcpyAsync(b.global, b.p, b.used, cudaMemcpyDeviceToDevice, s));
    b.held = COND_GLOBAL;
    return 0;
}

// Make block k hold override ov (nullptr: the lane's global values)
static int bind_block(b2sd_engine* h, int k, CondOverride* ov, cudaStream_t s) {
    auto& b = h->cond[k];
    const uint64_t want = ov ? ov->id : COND_GLOBAL;
    if (b.held == want) return 0;
    b.held = COND_UNKNOWN;
    if (ov) {
        CUDA_OK(cudaStreamWaitEvent(s, ov->ready, 0));
        CUDA_OK(cudaMemcpyAsync(b.p, ov->buf, b.used, cudaMemcpyDeviceToDevice, s));
        cudaEvent_t* use = nullptr;
        for (auto& u : ov->uses)
            if (u.first == s) use = &u.second;
        if (!use) {
            ov->uses.emplace_back(s, nullptr);
            use = &ov->uses.back().second;
            CUDA_OK(cudaEventCreateWithFlags(use, cudaEventDisableTiming));
        }
        CUDA_OK(cudaEventRecord(*use, s));
    } else {
        CUDA_OK(cudaMemcpyAsync(b.p, b.global, b.used, cudaMemcpyDeviceToDevice, s));
    }
    b.held = want;
    ++h->cond_binds;
    return 0;
}

// Make the blocks hold what `st` is stepped with (nullptr: a step without a state), before the frame program reads them
static int bind_conditioning(b2sd_engine* h, const b2sd_state* st, cudaStream_t s) {
    for (int k = 0; k < 2; ++k) {
        CondOverride* ov = st ? st->cond[k].get() : nullptr;
        if (ov && ov->store != h->ws->id) {
            b2_set_error("the state's own %s was computed with another weight store's parameters (a style's or its parent's): "
                         "set it again on an engine of this store", k == COND_PROMPT ? "prompt" : "timesteps");
            return -1;
        }
        TRY(bind_block(h, k, ov, s));
    }
    return 0;
}

static std::shared_ptr<CondPool> cond_pool(b2sd_engine* h) {
    std::shared_ptr<CondPool>& cp = h->ws->cond_pool;
    if (cp) return cp;
    auto p = std::make_shared<CondPool>();
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    cudaMemPoolProps props{};
    props.allocType = cudaMemAllocationTypePinned;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = dev;
    int no = 0;
    // Keep the memory of a few overrides across synchronisations (the default threshold, 0, hands freed memory back to the
    // driver at every one, and the next override maps it again inside cudaMallocFromPoolAsync); it is released with the pool.
    uint64_t keep = 4 * (uint64_t)(h->cond[COND_PROMPT].cap + h->cond[COND_TIME].cap);
    if (keep < (64ull << 20)) keep = 64ull << 20;   // the pool maps memory in chunks of tens of MiB
    if (e == cudaSuccess) e = cudaMemPoolCreate(&p->pool, &props);
    if (e == cudaSuccess) e = cudaMemPoolSetAttribute(p->pool, cudaMemPoolReuseAllowInternalDependencies, &no);
    if (e == cudaSuccess) e = cudaMemPoolSetAttribute(p->pool, cudaMemPoolAttrReleaseThreshold, &keep);
    if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&p->reaper, cudaStreamNonBlocking);
    if (e != cudaSuccess) {
        b2_set_error("conditioning override pool: %s", cudaGetErrorString(e));
        return nullptr;
    }
    cp = p;
    return cp;
}

// The prompt / time program has just computed `st`'s values into h's block k on s: copy them into a new override of the state
// (h's block holds it).  The override it replaces is freed after every copy out of it.
static int publish_override(b2sd_engine* h, b2sd_state* st, int k, cudaStream_t s, bool own_text = false) {
    static std::atomic<uint64_t> next_id{1};
    auto& b = h->cond[k];
    std::unique_ptr<CondOverride> ov(new CondOverride);
    ov->pool = cond_pool(h);
    if (!ov->pool) return -1;
    ov->id = next_id++;
    ov->store = h->ws->id;
    ov->own_text = own_text;
    ov->bytes = b.used;
    cudaError_t e = cudaEventCreateWithFlags(&ov->ready, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaMallocFromPoolAsync(&ov->buf, ov->bytes, ov->pool->pool, s);
    if (e == cudaSuccess) e = cudaMemcpyAsync(ov->buf, b.p, b.used, cudaMemcpyDeviceToDevice, s);
    if (ov->ready) {
        const cudaError_t er = cudaEventRecord(ov->ready, s);
        if (e == cudaSuccess) e = er;
    }
    if (e != cudaSuccess) {
        b2_set_error("conditioning override of %zu bytes: %s", ov->bytes, cudaGetErrorString(e));
        return -1;
    }
    b.held = ov->id;
    st->cond[k] = std::move(ov);
    return 0;
}

// ================================================================================================
extern "C" {

static int create_engine(const b2sd_config* cfg, std::shared_ptr<WeightStore> store, b2sd_handle* out);

int b2sd_create(const b2sd_config* cfg, b2sd_handle* out) { return create_engine(cfg, std::make_shared<WeightStore>(), out); }

/* A second engine over the SAME parameters (shared weight store): its own activations, stream state and CUDA graph, so two
 * frames can be in flight on two CUDA streams.  cfg may differ from the parent's in batch / size only. */
int b2sd_create_lane(b2sd_handle parent, const b2sd_config* cfg, b2sd_handle* out) {
    if (!parent) {
        b2_set_error("b2sd_create_lane: null parent");
        return -1;
    }
    b2sd_config c = cfg ? *cfg : parent->cfg;
    c.controlnet = parent->cfg.controlnet;   // a lane runs the parent's networks
    c.control_processor = parent->cfg.control_processor;
    memcpy(c.control_processor_more, parent->cfg.control_processor_more, sizeof(c.control_processor_more));
    c.vae = parent->cfg.vae;
    c.vae_scaling_factor = parent->cfg.vae_scaling_factor;
    c.ip_tokens = parent->cfg.ip_tokens;
    for (int i = 0; i < 4; ++i)
        if (c.block_out_channels[i] != parent->cfg.block_out_channels[i] || c.heads[i] != parent->cfg.heads[i] ||
            c.down_attn[i] != parent->cfg.down_attn[i]) {
            b2_set_error("b2sd_create_lane: the lane's architecture differs from its parent's");
            return -1;
        }
    if (create_engine(&c, parent->ws, out)) return -1;
    (*out)->concurrency = parent->concurrency > 1 ? parent->concurrency : 2;
    return 0;
}

static int create_engine(const b2sd_config* cfg, std::shared_ptr<WeightStore> store, b2sd_handle* out) {
    if (!cfg || !out) {
        b2_set_error("b2sd_create: null argument");
        return -1;
    }
    if (cfg->height % 64 || cfg->width % 64 || cfg->batch < 1 || cfg->batch > 16) {
        b2_set_error("b2sd_create: height/width must be multiples of 64, 1 <= batch <= 16 (got %dx%d, %d)",
                     cfg->height, cfg->width, cfg->batch);
        return -1;
    }
    for (int i = 0; i < 4; ++i) {
        if (cfg->block_out_channels[i] % 64 || cfg->heads[i] < 1 || cfg->block_out_channels[i] % cfg->heads[i]) {
            b2_set_error("b2sd_create: block_out_channels must be multiples of 64 and divisible by heads");
            return -1;
        }
    }
    if (cfg->cross_attention_dim % 64) {
        b2_set_error("b2sd_create: cross_attention_dim must be a multiple of 64");
        return -1;
    }
    if (cfg->controlnet < 0 || cfg->controlnet > B2SD_MAX_CONTROLNETS) {
        b2_set_error("b2sd_create: controlnet must be 0..%d (got %d)", B2SD_MAX_CONTROLNETS, cfg->controlnet);
        return -1;
    }
    const auto edge_processor = [](int p) { return p == B2SD_CONTROL_HED || p == B2SD_CONTROL_CANNY; };
    if (cfg->control_processor != B2SD_CONTROL_FRAME && (!edge_processor(cfg->control_processor) || !cfg->controlnet)) {
        b2_set_error("b2sd_create: control_processor must be 0 (the frame), 1 (HED) or 2 (Canny), the last two with a ControlNet "
                     "(got %d)", cfg->control_processor);
        return -1;
    }
    for (int i = 1; i < B2SD_MAX_CONTROLNETS; ++i) {
        const int p = cfg->control_processor_more[i - 1];
        if (p != B2SD_CONTROL_FRAME && (!edge_processor(p) || i >= cfg->controlnet)) {
            b2_set_error("b2sd_create: control_processor_more[%d] must be 0 (the frame), 1 (HED) or 2 (Canny), the last two with a "
                         "ControlNet %d (got %d)", i - 1, i, p);
            return -1;
        }
    }
    if (cfg->vae != B2SD_VAE_TINY && cfg->vae != B2SD_VAE_KL) {
        b2_set_error("b2sd_create: vae must be 0 (TAESD) or 1 (AutoencoderKL) (got %d)", cfg->vae);
        return -1;
    }
    if (!(cfg->vae_scaling_factor >= 0.f)) {
        b2_set_error("b2sd_create: vae_scaling_factor must be >= 0 (0 = 0.18215)");
        return -1;
    }
    if (cfg->ip_tokens < 0 || cfg->ip_tokens > ATTN_IP_KEYS) {
        b2_set_error("b2sd_create: ip_tokens must be 0 (no image prompts) or 1..%d (got %d)", ATTN_IP_KEYS, cfg->ip_tokens);
        return -1;
    }
    int dev = 0;
    cudaDeviceProp prop;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaGetDeviceProperties(&prop, dev) != cudaSuccess) {
        b2_set_error("b2sd_create: no CUDA device (this library has no CPU path)");
        return -1;
    }
    if (prop.major != 9 || prop.minor != 0) {
        b2_set_error("b2sd_create: device sm_%d%d is not Hopper sm_90 (kernels are sm_90a only)", prop.major, prop.minor);
        return -1;
    }
    if (igemm_init() || attn_init() || tconv_init()) return -1;
    b2sd_engine* e = new b2sd_engine(std::move(store));
    if (e->ws->order.s) {
        e->state.set_order(e->ws->order.s, e->ws->order.pool);
        e->prog.set_order(e->ws->order.s, e->ws->order.pool);
    }
    e->cfg = *cfg;
    e->lh = cfg->height / 8;
    e->lw = cfg->width / 8;
    const int B = cfg->batch, C0 = cfg->block_out_channels[0];
    e->x_in.n = B; e->x_in.h = e->lh; e->x_in.w = e->lw; e->x_in.c = 4; e->x_in.ld = 4;
    e->x_in.p = static_cast<__half*>(e->state.alloc((size_t)e->x_in.elems() * 2));
    e->noise = static_cast<__half*>(e->state.alloc((size_t)e->x_in.elems() * 2));
    e->coef = static_cast<float*>(e->state.alloc(4 * B * sizeof(float)));
    e->tsteps = static_cast<float*>(e->state.alloc(B * sizeof(float)));
    e->ctx = static_cast<__half*>(e->state.alloc((size_t)cfg->ctx_tokens * cfg->cross_attention_dim * 2));
    e->temb_sin = static_cast<float*>(e->state.alloc((size_t)B * C0 * sizeof(float)));
    e->temb_h = static_cast<float*>(e->state.alloc((size_t)B * 4 * C0 * sizeof(float)));
    e->temb = static_cast<float*>(e->state.alloc((size_t)B * 4 * C0 * sizeof(float)));
    bool cn_ok = true;
    for (int i = 0; i < cfg->controlnet; ++i) {
        e->cn_temb_h[i] = static_cast<float*>(e->state.alloc((size_t)B * 4 * C0 * sizeof(float)));
        e->cn_temb[i] = static_cast<float*>(e->state.alloc((size_t)B * 4 * C0 * sizeof(float)));
        cn_ok = cn_ok && e->cn_temb_h[i] && e->cn_temb[i];
    }
    for (auto& row : e->cn_scale_global) std::fill(row, row + 16, 1.f);
    e->gn_ws = static_cast<float*>(e->state.alloc(groupnorm_partial_floats(B, cfg->norm_groups) * sizeof(float)));
    e->tile_counters = static_cast<int*>(e->state.alloc(65536 * sizeof(int)));
    if (e->tile_counters) cudaMemset(e->tile_counters, 0, 65536 * sizeof(int));
    e->ctx_global = static_cast<__half*>(e->state.alloc((size_t)cfg->ctx_tokens * cfg->cross_attention_dim * 2));
    e->tsteps_global = static_cast<float*>(e->state.alloc(B * sizeof(float)));
    if (cfg->ip_tokens) {
        const size_t ip_bytes = (size_t)ATTN_IP_KEYS * cfg->cross_attention_dim * 2;
        e->ip_tok = static_cast<__half*>(e->state.alloc(ip_bytes));
        e->ip_tok_global = static_cast<__half*>(e->state.alloc(ip_bytes));
        if (!e->ip_tok || !e->ip_tok_global || cudaMemset(e->ip_tok, 0, ip_bytes) != cudaSuccess ||
            cudaMemset(e->ip_tok_global, 0, ip_bytes) != cudaSuccess) {
            b2_set_error("b2sd_create: cudaMalloc failed");
            delete e;
            return -1;
        }
    }
    if (!e->x_in.p || !e->noise || !e->coef || !e->tsteps || !e->ctx || !e->temb || !e->gn_ws || !e->ctx_global || !e->tsteps_global ||
        !cn_ok) {
        b2_set_error("b2sd_create: cudaMalloc failed");
        delete e;
        return -1;
    }
    *out = e;
    return 0;
}

int b2sd_destroy(b2sd_handle h) {
    if (h) {
        cudaDeviceSynchronize();
        delete h;
    }
    return 0;
}

// Parameters whose raw layout no kernel reads: they are re-laid-out once by pack_conv / pack_rows / small_w.
static bool is_pack_only(const std::string& key, const int64_t* shape, int ndim) {
    auto has = [&](const char* t) { return key.find(t) != std::string::npos; };
    if (ndim == 4 && shape[2] == 3) return true;                       // every 3x3 convolution (incl. the Cin <= 4 ones)
    if (ndim == 4 && has("conv_shortcut.weight")) return true;         // packed into the conv2 rows
    if (ndim == 4 && (has("controlnet_down_blocks.") || has("controlnet_mid_block."))) return true;   // ControlNet zero convs
    if (ndim == 2 && (has(".to_q.weight") || has(".to_k.weight") || has(".to_v.weight"))) return true;   // per-head gather
    if (ndim == 2 && has("ff.net.0.proj.weight")) return true;         // GEGLU value/gate interleave
    return false;
}

int b2sd_load_tensor(b2sd_handle h, const char* key, const void* ptr, int dtype, const int64_t* shape, int ndim) {
    if (!h || !key || !ptr || ndim < 1 || ndim > 4) {
        b2_set_error("b2sd_load_tensor: bad argument");
        return -1;
    }
    Raw r;
    r.shape.assign(shape, shape + ndim);
    const long n = r.numel();
    if (h->raw_released) {
        b2_set_error("b2sd_load_tensor(%s): the pack-only raw weights were released after b2sd_prepare; create a new engine to "
                     "load different parameters (or set B2_KEEP_RAW=1 before the first prepare)", key);
        return -1;
    }
    if (h->ws->live_ready) {
        b2_set_error("b2sd_load_tensor(%s): the engine's parameters are live (b2sd_set_live_params) and prepared; change them "
                     "with b2sd_apply_lora", key);
        return -1;
    }
    r.pack_only = is_pack_only(key, shape, ndim);
    auto old = h->raw.find(key);
    if (old != h->raw.end()) {
        // Reload of a parameter (e.g. a LoRA swap): everything derived from the old values is stale.  The packed / fp32
        // caches are keyed by parameter name, so drop them all (they are rebuilt by the next b2sd_prepare); a same-shape
        // reload overwrites the device copy in place instead of growing the bump arena.
        h->packed.clear(); h->packed_bytes.clear();
        h->fvec.clear(); h->fvec_bytes.clear();
        if (old->second.shape == r.shape) r.p = old->second.p;
        for (auto it = h->raw.begin(); it != h->raw.end();) it = it->second.derived ? h->raw.erase(it) : std::next(it);
    }
    if (!r.p) r.p = static_cast<__half*>((r.pack_only ? h->raw_only : h->weights).alloc((size_t)n * 2));
    if (!r.p) {
        b2_set_error("b2sd_load_tensor: cudaMalloc failed for %s", key);
        return -1;
    }
    if (dtype == 0) {
        CUDA_OK(cudaMemcpy(r.p, ptr, (size_t)n * 2, cudaMemcpyDefault));
    } else if (dtype == 1) {
        float* tmp = nullptr;
        CUDA_OK(cudaMalloc(&tmp, (size_t)n * 4));
        cudaError_t e1 = cudaMemcpy(tmp, ptr, (size_t)n * 4, cudaMemcpyDefault);
        int rc = (e1 == cudaSuccess) ? cast_f32_to_f16_launch(tmp, r.p, n, 0) : -1;
        cudaDeviceSynchronize();
        cudaFree(tmp);
        if (rc) {
            b2_set_error("b2sd_load_tensor: upload of %s failed", key);
            return -1;
        }
    } else {
        b2_set_error("b2sd_load_tensor: dtype %d", dtype);
        return -1;
    }
    // 1-D parameters get a host copy (fused fp32 vectors); so do HED's [1,3,1,1] offset and [1,C,1,1] projections, read as vectors
    const std::string k(key);
    const bool hed_vec = k == "hed.norm" || (k.compare(0, 4, "hed.") == 0 && k.size() > 18 && k.compare(k.size() - 18, 18, ".projection.weight") == 0);
    if (ndim == 1 || hed_vec) {
        std::vector<__half> hh(n);
        CUDA_OK(cudaMemcpy(hh.data(), r.p, (size_t)n * 2, cudaMemcpyDeviceToHost));
        r.host.resize(n);
        for (long i = 0; i < n; ++i) r.host[i] = __half2float(hh[i]);
    }
    h->raw[key] = std::move(r);
    h->built = false;
    return 0;
}

// TimestepEmbedding of the UNet (and of the ControlNet, from the same sinusoidal features): the launches that precede prog_time,
// with their launch records
static int time_embedding_ops(b2sd_handle h, std::vector<Op>* ops) {
    const int B = h->cfg.batch, C0 = h->cfg.block_out_channels[0], TD = 4 * C0;
    const float* t = h->tsteps;
    float* sin_ = h->temb_sin;
    b2sd_launch_record r{};
    r.kind = B2SD_LAUNCH_TIMESTEP_EMBEDDING;
    r.timestep_embedding = b2sd_timestep_embedding_args{t, sin_, B, C0};
    ops->push_back(Op([=](cudaStream_t st) { return timestep_embedding_launch(t, sin_, B, C0, st); }, "timestep_embedding", r));
    auto embed = [&](const std::string& p, float* hid, float* out) {
        const Raw* w1 = h->get(p + "time_embedding.linear_1.weight");
        const Raw* w2 = h->get(p + "time_embedding.linear_2.weight");
        const float* b1 = h->vec({p + "time_embedding.linear_1.bias"});
        const float* b2v = h->vec({p + "time_embedding.linear_2.bias"});
        if (!w1 || !w2 || !b1 || !b2v) return -1;
        const __half *w1p = w1->p, *w2p = w2->p;
        ops->push_back(Op([=](cudaStream_t st) { return small_linear_launch(sin_, C0, w1p, b1, hid, TD, B, TD, C0, 0, st); },
                          p + "time_embedding.linear_1", small_linear_record(sin_, C0, w1p, b1, hid, TD, B, TD, C0, 0)));
        ops->push_back(Op([=](cudaStream_t st) { return small_linear_launch(hid, TD, w2p, b2v, out, TD, B, TD, TD, 1, st); },
                          p + "time_embedding.linear_2", small_linear_record(hid, TD, w2p, b2v, out, TD, B, TD, TD, 1)));
        return 0;
    };
    TRY(embed("", h->temb_h, h->temb));
    for (int i = 0; i < h->cfg.controlnet; ++i) TRY(embed(cn_prefix(i), h->cn_temb_h[i], h->cn_temb[i]));
    return 0;
}

// the time embeddings, then every resnet's projection
static int refresh_time(b2sd_handle h, cudaStream_t s) {
    std::vector<Op> ops;
    TRY(time_embedding_ops(h, &ops));
    TRY(h->run(ops, s));
    return h->run(h->prog_time, s);
}

// A UNet matrix a LoRA may re-fuse: a loaded (not derived) parameter without a sub-network prefix ("controlnet" covers every
// net's "controlnet." / "controlnet<i>."), 2-D or 4-D
static bool lora_target(const std::string& key, const Raw& r) {
    for (const char* pre : {"vae.", "controlnet", "hed."})
        if (key.compare(0, strlen(pre), pre) == 0) return false;
    if (key.find("_ip.weight") != std::string::npos) return false;   // IP-Adapter's to_k_ip / to_v_ip: styles share them
    return !r.derived && r.shape.size() >= 2;
}

// Live mode, after the first prepare: the raw copies of the pack-only UNet matrices are kept as their base values (the packed
// entries are rebuilt from them), and every UNet matrix a kernel reads raw gets a base copy beside it, so that its live copy
// can be re-fused at the address the frame program holds.
static int make_live_base(b2sd_handle h) {
    WeightStore& w = *h->ws;
    if (w.live_ready) return 0;
    for (auto& kv : w.raw) {
        if (kv.second.pack_only || !lora_target(kv.first, kv.second)) continue;
        const size_t bytes = (size_t)kv.second.numel() * 2;
        __half* b = static_cast<__half*>(w.base_arena.alloc(bytes));
        if (!b) return -1;
        CUDA_OK(cudaMemcpy(b, kv.second.p, bytes, cudaMemcpyDeviceToDevice));
        w.base[kv.first] = b;
    }
    w.live_ready = true;
    return 0;
}

// *p = v as a 4-byte memset node on s (cuMemsetD32Async: the value travels with the command, nothing host-side to keep alive)
static int set_int_async(int* p, int v, cudaStream_t s) {
    using MemsetD32 = CUresult (*)(CUdeviceptr, unsigned int, size_t, CUstream);
    static MemsetD32 fn = nullptr;
    if (!fn) {
        void* fp = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuMemsetD32Async", &fp, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess || !fp) {
            b2_set_error("cudaGetDriverEntryPoint(cuMemsetD32Async) failed");
            return -1;
        }
        fn = reinterpret_cast<MemsetD32>(fp);
    }
    const CUresult r = fn(reinterpret_cast<CUdeviceptr>(p), (unsigned int)v, 1, s);
    if (r != CUDA_SUCCESS) {
        b2_set_error("cuMemsetD32Async failed: %d", (int)r);
        return -1;
    }
    return 0;
}

// The image program on ip_tok, whose first n rows hold an image prompt's tokens (n = 0: none): every UNet cross-attention's
// image K / V^T (V^T times scale) and the token count the attention kernel reads, in the prompt block.  Nothing without
// ip_tokens.
static int run_image(b2sd_handle h, int n, float scale, cudaStream_t s) {
    if (!h->cfg.ip_tokens) return 0;
    h->ip_scale = scale;
    TRY(h->run(h->prog_image, s));
    return set_int_async(h->ip_count, n, s);
}

int b2sd_prepare(b2sd_handle h, const void* prompt_embeds, const float* timesteps, const float* coef,
                 const void* init_noise, void* stream) {
    if (!h || !prompt_embeds || !timesteps || !coef || !init_noise) {
        b2_set_error("b2sd_prepare: null argument");
        return -1;
    }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const int B = h->cfg.batch, lh = h->lh, lw = h->lw;
    for (int k = 0; k < 4; ++k)
        for (int i = 0; i < B; ++i) h->coef_host[k][i] = coef[k * B + i];
    CUDA_OK(cudaMemcpyAsync(h->coef, coef, 4 * B * sizeof(float), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaMemcpyAsync(h->tsteps, timesteps, B * sizeof(float), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaMemcpyAsync(h->ctx, prompt_embeds, (size_t)h->cfg.ctx_tokens * h->cfg.cross_attention_dim * 2,
                            cudaMemcpyHostToDevice, s));
    // init_noise NCHW -> NHWC (host side; once per prepare)
    {
        const __half* src = static_cast<const __half*>(init_noise);
        std::vector<__half> nhwc((size_t)B * lh * lw * 4);
        for (int b = 0; b < B; ++b)
            for (int c = 0; c < 4; ++c)
                for (int y = 0; y < lh; ++y)
                    for (int x = 0; x < lw; ++x)
                        nhwc[(((size_t)b * lh + y) * lw + x) * 4 + c] = src[(((size_t)b * 4 + c) * lh + y) * lw + x];
        CUDA_OK(cudaMemcpyAsync(h->noise, nhwc.data(), nhwc.size() * 2, cudaMemcpyHostToDevice, s));
        CUDA_OK(cudaStreamSynchronize(s));
    }
    // x_t_latent_buffer = zeros (StreamDiffusion.prepare); slot 0 is overwritten by every frame
    CUDA_OK(cudaMemsetAsync(h->x_in.p, 0, (size_t)h->x_in.elems() * 2, s));
    for (auto& c : h->ws->pending)   // a style's own UNet matrices start as the base values, before anything packs them
        CUDA_OK(cudaMemcpyAsync(c.dst, c.src, c.bytes, cudaMemcpyDeviceToDevice, s));
    h->ws->pending.clear();
    const size_t rebuilds = h->ws->rebuild.size();
    TRY(h->build_program(s));
    if (h->ws->rebuild.size() != rebuilds && !h->ws->fused.empty()) {
        // new packed entries (a lane with another weight layout) were made from the base values, not the fused ones
        b2_set_error("b2sd_prepare: this engine needs packed weights the store did not have when b2sd_apply_lora ran; prepare "
                     "every lane before the first b2sd_apply_lora, or apply the LoRAs again");
        return -1;
    }
    TRY(h->run(h->prog_prompt, s));
    TRY(run_image(h, h->ip_n_global, h->ip_scale_global, s));
    TRY(refresh_time(h, s));
    TRY(write_global_scales(h, s));
    CUDA_OK(cudaMemcpyAsync(h->ctx_global, h->ctx, (size_t)h->cfg.ctx_tokens * h->cfg.cross_attention_dim * 2,
                            cudaMemcpyDeviceToDevice, s));
    CUDA_OK(cudaMemcpyAsync(h->tsteps_global, h->tsteps, B * sizeof(float), cudaMemcpyDeviceToDevice, s));
    TRY(keep_global(h, COND_PROMPT, s));
    TRY(keep_global(h, COND_TIME, s));
    CUDA_OK(cudaStreamSynchronize(s));
    if (h->ws->live) return make_live_base(h);
    // Every pack-only parameter now exists in its kernel-native layout: drop the raw copies (about half of the UNet's
    // 1.73 GB).  Later prepares hit the packed caches and never touch them.
    static const bool keep_raw = getenv("B2_KEEP_RAW") != nullptr;
    if (!keep_raw && !h->raw_released) {
        for (auto& kv : h->raw)
            if (kv.second.pack_only) kv.second.p = nullptr;
        h->raw_only.release();
        h->raw_released = true;
    }
    return 0;
}

// ---- packed-weight blob (replaces the reference's TensorRT engine files, lib/wrapper.py:593-597, 896-910) -----------------
// Layout: "B2SDPACK" u32 version, b2sd_config, u32 count, then per entry
//   u8 kind (0 raw parameter, 1 packed fp16 matrix, 2 fp32 vector) | u32 name length | name | u32 ndim | i64 shape[ndim] |
//   u64 payload bytes (0 for a raw pack-only parameter: only its shape is needed) | payload
extern "C++" {
namespace {
struct BlobWriter {
    FILE* f;
    bool ok = true;
    void put(const void* p, size_t n) { if (ok && n && fwrite(p, 1, n, f) != n) ok = false; }
    template <class T> void pod(const T& v) { put(&v, sizeof(T)); }
    void str(const std::string& v) { pod((uint32_t)v.size()); put(v.data(), v.size()); }
};
struct BlobReader {
    FILE* f;
    bool ok = true;
    void get(void* p, size_t n) { if (ok && n && fread(p, 1, n, f) != n) ok = false; }
    template <class T> T pod() { T v{}; get(&v, sizeof(T)); return v; }
    std::string str() { uint32_t n = pod<uint32_t>(); if (!ok || n > 4096) { ok = false; return ""; } std::string v(n, 0); get(&v[0], n); return v; }
};
}  // namespace
}  // extern "C++"

int b2sd_export_packed(b2sd_handle h, const char* path) {
    if (!h || !h->built || !path) {
        b2_set_error("b2sd_export_packed: call b2sd_prepare first");
        return -1;
    }
    FILE* f = fopen(path, "wb");
    if (!f) {
        b2_set_error("b2sd_export_packed: cannot open %s", path);
        return -1;
    }
    BlobWriter w{f};
    w.put("B2SDPACK", 8);
    // 5: b2sd_config carries `control_processor_more` (4: up to `ip_tokens`, 3: up to `vae_scaling_factor`, 2: up to
    // `control_processor`; 1-4 still load)
    w.pod((uint32_t)5);
    b2sd_config cfg = h->cfg;
    cfg.batch = 0; cfg.height = 0; cfg.width = 0; cfg.use_cuda_graph = 0; cfg.do_add_noise = 0;   // the blob is independent of these
    w.pod(cfg);
    w.pod((uint32_t)(h->raw.size() + h->packed_bytes.size() + h->fvec_bytes.size()));
    std::vector<char> host;
    auto payload = [&](const void* dptr, size_t bytes) {
        w.pod((uint64_t)bytes);
        if (!bytes) return true;
        host.resize(bytes);
        if (cudaMemcpy(host.data(), dptr, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) return false;
        w.put(host.data(), bytes);
        return true;
    };
    bool copy_ok = true;
    for (auto& kv : h->raw) {
        const Raw& r = kv.second;
        w.pod((uint8_t)0); w.str(kv.first);
        w.pod((uint32_t)r.shape.size());
        for (auto d : r.shape) w.pod((int64_t)d);
        copy_ok &= payload(r.p, (r.pack_only || !r.p) ? 0 : (size_t)r.numel() * 2);
    }
    for (auto& kv : h->packed_bytes) {
        w.pod((uint8_t)1); w.str(kv.first); w.pod((uint32_t)0);
        copy_ok &= payload(h->packed[kv.first], kv.second);
    }
    for (auto& kv : h->fvec_bytes) {
        w.pod((uint8_t)2); w.str(kv.first); w.pod((uint32_t)0);
        copy_ok &= payload(h->fvec[kv.first], kv.second);
    }
    const bool ok = w.ok && copy_ok && fclose(f) == 0;
    if (!ok) {
        b2_set_error("b2sd_export_packed: write to %s failed", path);
        remove(path);
        return -1;
    }
    return 0;
}

int b2sd_import_packed(b2sd_handle h, const char* path) {
    if (!h || !path) {
        b2_set_error("b2sd_import_packed: null argument");
        return -1;
    }
    if (!h->raw.empty()) {
        b2_set_error("b2sd_import_packed: the engine already holds parameters");
        return -1;
    }
    if (h->ws->live) {
        b2_set_error("b2sd_import_packed: the engine's parameters are live (b2sd_set_live_params): a blob does not carry the "
                     "base parameters they are re-fused from; load them with b2sd_load_tensor");
        return -1;
    }
    FILE* f = fopen(path, "rb");
    if (!f) {
        b2_set_error("b2sd_import_packed: cannot open %s", path);
        return -1;
    }
    BlobReader rd{f};
    char magic[8];
    rd.get(magic, 8);
    const uint32_t version = rd.pod<uint32_t>();
    // version 1 blobs predate the ControlNet fields at the end of b2sd_config: they hold no ControlNet (both fields 0);
    // version 2 blobs end b2sd_config before `vae`: they hold TAESD (vae = 0); version 3 blobs before `ip_tokens`: no IP-Adapter;
    // version 4 blobs before `control_processor_more`: at most one ControlNet
    b2sd_config cfg{};
    if (version == 1) rd.get(&cfg, offsetof(b2sd_config, controlnet));
    else if (version == 2) rd.get(&cfg, offsetof(b2sd_config, vae));
    else if (version == 3) rd.get(&cfg, offsetof(b2sd_config, ip_tokens));
    else if (version == 4) rd.get(&cfg, offsetof(b2sd_config, control_processor_more));
    else cfg = rd.pod<b2sd_config>();
    if (rd.ok && version >= 1 && version <= 5 && (cfg.ip_tokens != 0) != (h->cfg.ip_tokens != 0)) {
        fclose(f);
        b2_set_error("b2sd_import_packed: %s was packed %s an IP-Adapter and this engine has %s", path,
                     cfg.ip_tokens ? "with" : "without", h->cfg.ip_tokens ? "one" : "none");
        return -1;
    }
    bool same = rd.ok && memcmp(magic, "B2SDPACK", 8) == 0 && version >= 1 && version <= 5 && cfg.cross_attention_dim == h->cfg.cross_attention_dim &&
                cfg.layers_per_block == h->cfg.layers_per_block && cfg.norm_groups == h->cfg.norm_groups && cfg.ctx_tokens == h->cfg.ctx_tokens &&
                cfg.controlnet == h->cfg.controlnet && cfg.control_processor == h->cfg.control_processor &&
                memcmp(cfg.control_processor_more, h->cfg.control_processor_more, sizeof(cfg.control_processor_more)) == 0 &&
                cfg.vae == h->cfg.vae &&
                (cfg.vae != B2SD_VAE_KL || cfg.vae_scaling_factor == h->cfg.vae_scaling_factor);
    for (int i = 0; i < 4 && same; ++i)
        same = cfg.block_out_channels[i] == h->cfg.block_out_channels[i] && cfg.heads[i] == h->cfg.heads[i] && cfg.down_attn[i] == h->cfg.down_attn[i];
    if (!same) {
        fclose(f);
        b2_set_error("b2sd_import_packed: %s is not a packed-weight blob of this architecture", path);
        return -1;
    }
    const uint32_t count = rd.pod<uint32_t>();
    std::vector<char> host;
    for (uint32_t i = 0; i < count && rd.ok; ++i) {
        const uint8_t kind = rd.pod<uint8_t>();
        const std::string name = rd.str();
        const uint32_t ndim = rd.pod<uint32_t>();
        Raw r;
        for (uint32_t d = 0; d < ndim && d < 8; ++d) r.shape.push_back(rd.pod<int64_t>());
        const uint64_t bytes = rd.pod<uint64_t>();
        if (!rd.ok || bytes > ((uint64_t)1 << 32)) { rd.ok = false; break; }
        void* dptr = nullptr;
        if (bytes) {
            host.resize(bytes);
            rd.get(host.data(), bytes);
            dptr = h->weights.alloc(bytes);
            if (!rd.ok || !dptr || cudaMemcpy(dptr, host.data(), bytes, cudaMemcpyHostToDevice) != cudaSuccess) { rd.ok = false; break; }
        }
        if (kind == 0) {
            r.p = static_cast<__half*>(dptr);
            r.pack_only = bytes == 0;
            if (ndim == 1 && bytes) {
                const __half* hp = reinterpret_cast<const __half*>(host.data());
                r.host.resize(bytes / 2);
                for (size_t k = 0; k < r.host.size(); ++k) r.host[k] = __half2float(hp[k]);
            }
            h->raw[name] = std::move(r);
        } else if (kind == 1) {
            h->packed[name] = static_cast<__half*>(dptr);
            h->packed_bytes[name] = bytes;
        } else if (kind == 2) {
            h->fvec[name] = static_cast<float*>(dptr);
            h->fvec_bytes[name] = bytes;
        } else {
            rd.ok = false;
        }
    }
    fclose(f);
    if (!rd.ok) {
        b2_set_error("b2sd_import_packed: %s is truncated or corrupt", path);
        return -1;
    }
    h->raw_released = true;   // there never was a raw copy of the pack-only parameters
    h->imported = true;
    h->built = false;
    return 0;
}

int b2sd_set_prompt_embeds(b2sd_handle h, const void* prompt_embeds, void* stream) {
    if (!h || !h->built) {
        b2_set_error("b2sd_set_prompt_embeds: call b2sd_prepare first");
        return -1;
    }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const size_t bytes = (size_t)h->cfg.ctx_tokens * h->cfg.cross_attention_dim * 2;
    CUDA_OK(cudaMemcpyAsync(h->ctx, prompt_embeds, bytes, cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaStreamSynchronize(s));
    CUDA_OK(cudaMemcpyAsync(h->ctx_global, h->ctx, bytes, cudaMemcpyDeviceToDevice, s));
    if (h->cfg.ip_tokens) TRY(bind_block(h, COND_PROMPT, nullptr, s));   // keep the global image part of the block
    h->cond[COND_PROMPT].held = COND_UNKNOWN;
    TRY(h->run(h->prog_prompt, s));
    return keep_global(h, COND_PROMPT, s);
}

int b2sd_set_timesteps(b2sd_handle h, const float* timesteps, void* stream) {
    if (!h || !h->built) {
        b2_set_error("b2sd_set_timesteps: call b2sd_prepare first");
        return -1;
    }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    CUDA_OK(cudaMemcpyAsync(h->tsteps, timesteps, h->cfg.batch * sizeof(float), cudaMemcpyHostToDevice, s));
    CUDA_OK(cudaStreamSynchronize(s));
    CUDA_OK(cudaMemcpyAsync(h->tsteps_global, h->tsteps, h->cfg.batch * sizeof(float), cudaMemcpyDeviceToDevice, s));
    if (h->cn_scale) TRY(bind_block(h, COND_TIME, nullptr, s));   // keep the global ControlNet scales of the block
    h->cond[COND_TIME].held = COND_UNKNOWN;
    TRY(refresh_time(h, s));
    return keep_global(h, COND_TIME, s);
}

// The single-net form of a control-scale call refuses an engine with several nets
static int refuse_multi(const char* fn, b2sd_handle h) {
    if (h && h->cfg.controlnet > 1) {
        b2_set_error("%s: the engine has %d ControlNets; set their scales with %ss", fn, h->cfg.controlnet, fn);
        return -1;
    }
    return 0;
}

static int set_control_scales(const char* fn, b2sd_handle h, const float* per_net_slot, void* stream) {
    if (!h || !h->built || !per_net_slot) {
        b2_set_error("%s: null argument, or b2sd_prepare not called", fn);
        return -1;
    }
    if (!h->cn_scale) {
        b2_set_error("%s: the engine was created without a ControlNet (b2sd_config.controlnet = 0)", fn);
        return -1;
    }
    const int B = h->cfg.batch;
    for (int i = 0; i < h->cfg.controlnet; ++i)
        for (int k = 0; k < B; ++k)
            if (!isfinite(per_net_slot[i * B + k])) {
                if (h->cfg.controlnet == 1)
                    b2_set_error("%s: the scale of slot %d is not finite (%f)", fn, k, (double)per_net_slot[k]);
                else
                    b2_set_error("%s: the scale of net %d, slot %d is not finite (%f)", fn, i, k, (double)per_net_slot[i * B + k]);
                return -1;
            }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    for (int i = 0; i < h->cfg.controlnet; ++i) memcpy(h->cn_scale_global[i], per_net_slot + i * B, B * sizeof(float));
    TRY(bind_block(h, COND_TIME, nullptr, s));   // keep the global time biases of the block
    h->cond[COND_TIME].held = COND_UNKNOWN;
    TRY(write_global_scales(h, s));
    return keep_global(h, COND_TIME, s);
}

int b2sd_set_control_scale(b2sd_handle h, const float* scale_per_slot, void* stream) {
    TRY(refuse_multi("b2sd_set_control_scale", h));
    return set_control_scales("b2sd_set_control_scale", h, scale_per_slot, stream);
}

int b2sd_set_control_scales(b2sd_handle h, const float* per_net_slot, void* stream) {
    return set_control_scales("b2sd_set_control_scales", h, per_net_slot, stream);
}

// ---- live parameters ------------------------------------------------------------------------------------------------------
int b2sd_set_live_params(b2sd_handle h, int on) {
    if (!h) {
        b2_set_error("b2sd_set_live_params: null handle");
        return -1;
    }
    WeightStore& w = *h->ws;
    if (w.raw_released || w.imported || w.live_ready) {
        b2_set_error("b2sd_set_live_params: call it before the first b2sd_prepare of the weight store, on parameters loaded with "
                     "b2sd_load_tensor");
        return -1;
    }
    w.live = on != 0;
    return 0;
}

static size_t align256(size_t b) { return (b + 255) & ~size_t(255); }

int b2sd_apply_lora(b2sd_handle h, int n, const b2sd_lora_factor* f, void* stream) {
    if (!h || n < 0 || (n > 0 && !f)) {
        b2_set_error("b2sd_apply_lora: bad argument");
        return -1;
    }
    WeightStore& w = *h->ws;
    if (!w.live || !w.live_ready) {
        b2_set_error("b2sd_apply_lora: the weight store is not live (b2sd_set_live_params before the first b2sd_prepare)");
        return -1;
    }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    // ---- validate everything before the first device operation
    struct Job { Raw* r = nullptr; long rows = 0, cols = 0; std::vector<const b2sd_lora_factor*> fs; };
    std::map<std::string, Job> jobs;
    size_t a_bytes = 0, b_bytes = 0, tmp_bytes = 0;
    for (int i = 0; i < n; ++i) {
        const b2sd_lora_factor& fc = f[i];
        auto it = fc.key ? w.raw.find(fc.key) : w.raw.end();
        if (it == w.raw.end() || !lora_target(it->first, it->second)) {
            b2_set_error("b2sd_apply_lora: factor %d: '%s' is not a UNet weight matrix of this engine", i, fc.key ? fc.key : "(null)");
            return -1;
        }
        if (!fc.up || !fc.down || fc.rank < 1 || fc.rank > 4096 || (fc.dtype != 0 && fc.dtype != 1) || !isfinite(fc.scale)) {
            b2_set_error("b2sd_apply_lora: factor %d (%s): null factor, rank %d outside 1..4096, dtype %d or a non-finite scale", i,
                         fc.key, fc.rank, fc.dtype);
            return -1;
        }
        Job& j = jobs[it->first];
        j.r = &it->second;
        j.rows = it->second.shape[0];
        j.cols = it->second.numel() / j.rows;
        j.fs.push_back(&fc);
        const size_t kp = (size_t)((fc.dtype ? 3 : 1) * fc.rank + IG_BK - 1) / IG_BK * IG_BK;
        a_bytes = std::max(a_bytes, align256(j.rows * kp * 2));
        b_bytes = std::max(b_bytes, align256(j.cols * kp * 2));
        tmp_bytes = std::max(tmp_bytes, align256((size_t)j.rows * j.cols * 2));
    }
    // the keys that change: listed ones, and those the previous call fused that now revert to their base
    std::map<std::string, bool> touched;   // key -> listed
    for (auto& kv : jobs) touched[kv.first] = true;
    for (auto& k : w.fused) touched.emplace(k, false);
    // packed entries to rebuild, and the fused matrices each needs at once
    std::vector<WeightStore::Rebuild*> entries;
    size_t slot_bytes = 0;
    for (auto& kv : w.rebuild) {
        size_t need = 0;
        bool hit = false;
        for (auto& k : kv.second.keys) {
            auto t = touched.find(k);
            if (t == touched.end()) continue;
            hit = true;
            if (t->second) need += align256((size_t)jobs[k].rows * jobs[k].cols * 2);
        }
        if (hit) entries.push_back(&kv.second);
        slot_bytes = std::max(slot_bytes, need);
    }
    // ---- scratch: [up operand | down operand | two chain buffers | fused matrices of one entry]
    const size_t need = a_bytes + b_bytes + 2 * tmp_bytes + slot_bytes;
    if (need > w.scratch_cap) {
        if (w.scratch) CUDA_OK(cudaFreeAsync(w.scratch, s));
        w.scratch = nullptr;
        w.scratch_cap = 0;
        CUDA_OK(w.order.pool ? cudaMallocFromPoolAsync(&w.scratch, need, w.order.pool, s) : cudaMallocAsync(&w.scratch, need, s));
        w.scratch_cap = need;
    }
    char* sp = static_cast<char*>(w.scratch);
    __half* opa = reinterpret_cast<__half*>(sp);
    __half* opb = reinterpret_cast<__half*>(sp + a_bytes);
    __half* tmp[2] = {reinterpret_cast<__half*>(sp + a_bytes + b_bytes), reinterpret_cast<__half*>(sp + a_bytes + b_bytes + tmp_bytes)};
    char* slots = sp + a_bytes + b_bytes + 2 * tmp_bytes;
    // from here on a failure leaves any touched key possibly fused: the next call restores all of them
    std::vector<std::string> now;
    for (auto& kv : touched) now.push_back(kv.first);
    w.fused = now;

    // out = base + sum of the key's deltas in order, rounded to fp16 after each: one igemm per factor, M = rows, N = cols,
    // K = rank (three parts for fp32 factors) zero-padded to the K block, epilogue scale * acc + residual
    auto fuse = [&](const Job& j, const __half* base, __half* out) -> int {
        const __half* prev = base;
        for (size_t i = 0; i < j.fs.size(); ++i) {
            const b2sd_lora_factor& fc = *j.fs[i];
            __half* dst = i + 1 == j.fs.size() ? out : tmp[i & 1];
            const int kp = ((fc.dtype ? 3 : 1) * fc.rank + IG_BK - 1) / IG_BK * IG_BK;
            TRY(lora_factor_launch(fc.up, fc.dtype, j.rows, fc.rank, fc.rank, 1, 2, opa, kp, s));     // up[r][k]
            TRY(lora_factor_launch(fc.down, fc.dtype, j.cols, fc.rank, 1, j.cols, 4, opb, kp, s));    // down[k][c], transposed
            IgemmDesc d{};
            d.nseg = 1; d.src[0] = ActView{opa, 1, 1, (int)j.rows, kp, kp}; d.ntap[0] = 1;
            d.w = opb; d.w_rows = (int)j.cols; d.w_ld = kp; d.stride = 1;
            d.Nb = 1; d.Ho = 1; d.Wo = (int)j.rows;
            d.epi.out = dst; d.epi.ldc = (int)j.cols;
            d.epi.res = prev; d.epi.ldr = (int)j.cols;
            d.epi.acc_scale = fc.scale; d.epi.res_scale = 1.f;
            d.epi.n_valid = (int)j.cols;
            IgemmPlan plan;
            TRY(igemm_plan(d, &plan));
            TRY(igemm_launch(plan, s));
            prev = dst;
        }
        return 0;
    };
    // matrices the kernels read raw: fused in place (the frame program holds their address), or copied back from the base
    for (auto& kv : touched) {
        Raw& r = w.raw[kv.first];
        if (r.pack_only) continue;
        __half* base = w.base[kv.first];
        if (kv.second) TRY(fuse(jobs[kv.first], base, r.p));
        else CUDA_OK(cudaMemcpyAsync(r.p, base, (size_t)r.numel() * 2, cudaMemcpyDeviceToDevice, s));
    }
    // packed entries: rebuilt in place from the fused matrices of their listed keys and the base of the others
    for (WeightStore::Rebuild* e : entries) {
        size_t off = 0;
        w.src_override.clear();
        for (auto& k : e->keys) {
            auto t = touched.find(k);
            if (t == touched.end() || !t->second || w.src_override.count(k)) continue;
            __half* out = reinterpret_cast<__half*>(slots + off);
            off += align256((size_t)jobs[k].rows * jobs[k].cols * 2);
            TRY(fuse(jobs[k], w.raw[k].p, out));
            w.src_override[k] = out;
        }
        const int rc = e->fn(s);
        w.src_override.clear();
        TRY(rc);
    }
    now.clear();
    for (auto& kv : jobs) now.push_back(kv.first);
    w.fused = now;
    return 0;
}

int b2sd_refresh_conditioning(b2sd_handle h, void* stream) {
    if (!h || !h->built) {
        b2_set_error("b2sd_refresh_conditioning: call b2sd_prepare first");
        return -1;
    }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    CUDA_OK(cudaMemcpyAsync(h->ctx, h->ctx_global, (size_t)h->cfg.ctx_tokens * h->cfg.cross_attention_dim * 2,
                            cudaMemcpyDeviceToDevice, s));
    CUDA_OK(cudaMemcpyAsync(h->tsteps, h->tsteps_global, h->cfg.batch * sizeof(float), cudaMemcpyDeviceToDevice, s));
    h->cond[COND_PROMPT].held = COND_UNKNOWN;
    h->cond[COND_TIME].held = COND_UNKNOWN;
    TRY(write_global_scales(h, s));
    TRY(h->run(h->prog_prompt, s));
    TRY(run_image(h, h->ip_n_global, h->ip_scale_global, s));
    TRY(refresh_time(h, s));
    TRY(keep_global(h, COND_PROMPT, s));
    return keep_global(h, COND_TIME, s);
}

// ---- styles ---------------------------------------------------------------------------------------------------------------
// Whether a packed / fp32 cache entry is derived from a UNet matrix a LoRA may change (a style then needs its own copy)
static bool lora_derived(const WeightStore& w, std::string name) {
    auto rb = w.rebuild.find(name);
    if (rb == w.rebuild.end()) {   // the LayerNorm fold's column sums and biases are rebuilt with the gathered rows
        for (const char* suffix : {":cs", ":b"}) {
            const size_t n = strlen(suffix);
            if (name.size() > n && name.compare(name.size() - n, n, suffix) == 0) {
                rb = w.rebuild.find(name.substr(0, name.size() - n));
                break;
            }
        }
    }
    if (rb == w.rebuild.end()) return false;
    for (auto& k : rb->second.keys) {
        auto it = w.raw.find(k);
        if (it != w.raw.end() && lora_target(k, it->second)) return true;
    }
    return false;
}

int b2sd_create_style(b2sd_handle parent, b2sd_handle* out) {
    if (!parent || !out) {
        b2_set_error("b2sd_create_style: null argument");
        return -1;
    }
    // derive from the family's root: its base values are the ones every style reads
    std::shared_ptr<WeightStore> root = parent->ws->parent ? parent->ws->parent : parent->ws;
    if (!root->live || !root->live_ready) {
        b2_set_error("b2sd_create_style: the parent's weight store is not live and prepared (b2sd_set_live_params before its "
                     "first b2sd_prepare)");
        return -1;
    }
    auto st = std::make_shared<WeightStore>();
    st->parent = root;
    st->family = root->family;
    st->live = st->live_ready = true;
    {   // the style's own pool, which never makes an allocation wait for a free on another stream (as CondPool)
        int dev = 0, no = 0;
        cudaError_t e = cudaGetDevice(&dev);
        cudaMemPoolProps props{};
        props.allocType = cudaMemAllocationTypePinned;
        props.location.type = cudaMemLocationTypeDevice;
        props.location.id = dev;
        if (e == cudaSuccess) e = cudaMemPoolCreate(&st->order.pool, &props);
        if (e == cudaSuccess) e = cudaMemPoolSetAttribute(st->order.pool, cudaMemPoolReuseAllowInternalDependencies, &no);
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&st->order.s, cudaStreamNonBlocking);
        if (e != cudaSuccess) {
            b2_set_error("b2sd_create_style: %s", cudaGetErrorString(e));
            return -1;
        }
    }
    st->weights.set_order(st->order.s, st->order.pool);
    st->raw_only.set_order(st->order.s, st->order.pool);
    st->base_arena.set_order(st->order.s, st->order.pool);
    // Parameters: the raw map's entries point at the root's memory (its base values for the pack-only UNet matrices), except
    // the UNet matrices kernels read raw, which get copies of their own, filled with the base values by the first prepare.
    st->raw = root->raw;
    for (auto& kv : st->raw) {
        Raw& r = kv.second;
        if (r.pack_only || !lora_target(kv.first, r)) continue;
        auto base = root->base.find(kv.first);
        if (base == root->base.end()) {
            b2_set_error("b2sd_create_style: the parent's store has no base value of '%s'", kv.first.c_str());
            return -1;
        }
        const size_t bytes = (size_t)r.numel() * 2;
        __half* p = static_cast<__half*>(st->weights.alloc(bytes));
        if (!p) return -1;
        st->base[kv.first] = base->second;
        st->pending.push_back({p, base->second, bytes});
        r.p = p;
    }
    // Cache entries no UNet LoRA reaches are shared; the others are made by the style's first prepare, from its own parameters
    for (auto& kv : root->packed)
        if (!lora_derived(*root, kv.first)) {
            st->packed[kv.first] = kv.second;
            st->packed_bytes[kv.first] = root->packed_bytes.at(kv.first);
        }
    for (auto& kv : root->fvec)
        if (!lora_derived(*root, kv.first)) {
            st->fvec[kv.first] = kv.second;
            st->fvec_bytes[kv.first] = root->fvec_bytes.at(kv.first);
        }
    if (create_engine(&parent->cfg, st, out)) return -1;
    (*out)->concurrency = parent->concurrency;
    return 0;
}

int b2sd_release(b2sd_handle h, void* stream) {
    if (!h) return 0;
    const cudaStream_t order = h->ws->order.s;
    if (!order) {
        b2_set_error("b2sd_release: the engine's weight store is not a style (b2sd_create_style); use b2sd_destroy");
        return -1;
    }
    cudaEvent_t last = nullptr;
    cudaError_t e = cudaEventCreateWithFlags(&last, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventRecord(last, reinterpret_cast<cudaStream_t>(stream));
    if (e == cudaSuccess) e = cudaStreamWaitEvent(order, last, 0);
    if (last) cudaEventDestroy(last);
    if (e != cudaSuccess) {
        b2_set_error("b2sd_release: %s", cudaGetErrorString(e));
        return -1;
    }
    delete h;   // its memory, and its store's once no engine holds it, is freed on `order` after the work queued on `stream`
    return 0;
}

// ---- per-state conditioning --------------------------------------------------------------------------
// What every call that runs a state on an engine refuses
static int check_state(const char* fn, b2sd_handle h, const b2sd_state* state) {
    if (!h || !h->built || !state) {
        b2_set_error("%s: null argument, or b2sd_prepare not called", fn);
        return -1;
    }
    if (state->family != h->ws->family || state->batch != h->cfg.batch || state->height != h->cfg.height ||
        state->width != h->cfg.width) {
        b2_set_error("%s: the state was made for another weight store, batch or size (state: batch %d, %dx%d; "
                     "engine: batch %d, %dx%d)", fn, state->batch, state->height, state->width, h->cfg.batch, h->cfg.height,
                     h->cfg.width);
        return -1;
    }
    return 0;
}

// The prompt block a refresh of `st`'s text (own_text = false) or image part (own_text = true) starts from: the state's override
// if it was computed on h's store and, for an image refresh, from the state's own prompt embeddings; else nullptr, the lane's
// global values.  An override whose text part came from the global prompt is not kept: the global block is recomputed by
// every global refresh (a new prompt, a LoRA switch), the override's copy of it is not.  After a move to another store of the
// family the state's own prompt and image prompt are set again.
static CondOverride* prompt_base(b2sd_engine* h, b2sd_state* st, bool own_text) {
    CondOverride* ov = st->cond[COND_PROMPT].get();
    return ov && ov->store == h->ws->id && (ov->own_text || !own_text) ? ov : nullptr;
}

// The time block a refresh of `st`'s timesteps (control = false) or ControlNet scales (control = true) starts from, so that it
// keeps the other part: the state's override if it was computed on h's store and holds that part of its own; else nullptr, the
// lane's global values.  As for the prompt block, a part taken from the global values is not kept: the state's own
// settings are set again after a global refresh.
static CondOverride* time_base(b2sd_engine* h, b2sd_state* st, bool control) {
    CondOverride* ov = st->cond[COND_TIME].get();
    return ov && ov->store == h->ws->id && (control ? ov->own_time : ov->own_control) ? ov : nullptr;
}

// Run h's prompt (k = COND_PROMPT) or time refresh on s with `input` (device) in place of the global embeddings / timesteps,
// put the global ones back, and publish the block as the state's override.  Stream-ordered after the frames queued on s, and
// no host synchronisation: the refresh writes only h's block, which no other stream reads.
static int state_refresh(const char* fn, b2sd_handle h, b2sd_state* state, int k, const void* input, cudaStream_t s) {
    TRY(check_state(fn, h, state));
    if (!input) {
        b2_set_error("%s: null argument", fn);
        return -1;
    }
    void* dst = k == COND_PROMPT ? (void*)h->ctx : (void*)h->tsteps;
    const void* global = k == COND_PROMPT ? (const void*)h->ctx_global : (const void*)h->tsteps_global;
    const size_t bytes = k == COND_PROMPT ? (size_t)h->cfg.ctx_tokens * h->cfg.cross_attention_dim * 2
                                          : (size_t)h->cfg.batch * sizeof(float);
    // with image prompts the prompt program leaves the image part of the block alone: start from the state's block, so that
    // the state keeps its own image prompt
    if (k == COND_PROMPT && h->cfg.ip_tokens) TRY(bind_block(h, k, prompt_base(h, state, false), s));
    // with a ControlNet the time program leaves the ControlNet scales of the block alone: start from the state's block if it
    // holds the state's own scales
    CondOverride* tbase = k == COND_TIME && h->cn_scale ? time_base(h, state, false) : nullptr;
    if (k == COND_TIME && h->cn_scale) TRY(bind_block(h, k, tbase, s));
    h->cond[k].held = COND_UNKNOWN;
    CUDA_OK(cudaMemcpyAsync(dst, input, bytes, cudaMemcpyDeviceToDevice, s));
    const int rc = k == COND_PROMPT ? h->run(h->prog_prompt, s) : refresh_time(h, s);
    CUDA_OK(cudaMemcpyAsync(dst, global, bytes, cudaMemcpyDeviceToDevice, s));
    TRY(rc);
    TRY(publish_override(h, state, k, s, k == COND_PROMPT));
    if (k == COND_TIME) {
        state->cond[k]->own_time = true;
        state->cond[k]->own_control = tbase != nullptr;
    }
    return 0;
}

int b2sd_state_set_prompt_embeds(b2sd_handle h, b2sd_state_handle state, const void* prompt_embeds, void* stream) {
    return state_refresh("b2sd_state_set_prompt_embeds", h, state, COND_PROMPT, prompt_embeds,
                         reinterpret_cast<cudaStream_t>(stream));
}

int b2sd_state_set_timesteps(b2sd_handle h, b2sd_state_handle state, const float* timesteps, void* stream) {
    return state_refresh("b2sd_state_set_timesteps", h, state, COND_TIME, timesteps, reinterpret_cast<cudaStream_t>(stream));
}

static int state_set_control_scales(const char* fn, b2sd_handle h, b2sd_state* state, const float* scale_per_slot, void* stream) {
    TRY(check_state(fn, h, state));
    if (!scale_per_slot) {
        b2_set_error("%s: null argument", fn);
        return -1;
    }
    if (!h->cn_scale) {
        b2_set_error("%s: the engine was created without a ControlNet (b2sd_config.controlnet = 0)", fn);
        return -1;
    }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    CondOverride* base = time_base(h, state, true);   // the state's time biases: its own timesteps', or the global ones
    TRY(bind_block(h, COND_TIME, base, s));
    h->cond[COND_TIME].held = COND_UNKNOWN;
    CUDA_OK(cudaMemcpyAsync(h->cn_scale, scale_per_slot, (size_t)h->cfg.controlnet * h->cfg.batch * sizeof(float),
                            cudaMemcpyDeviceToDevice, s));
    TRY(publish_override(h, state, COND_TIME, s));
    state->cond[COND_TIME]->own_time = base != nullptr;
    state->cond[COND_TIME]->own_control = true;
    return 0;
}

int b2sd_state_set_control_scale(b2sd_handle h, b2sd_state_handle state, const float* scale_per_slot, void* stream) {
    TRY(refuse_multi("b2sd_state_set_control_scale", h));
    return state_set_control_scales("b2sd_state_set_control_scale", h, state, scale_per_slot, stream);
}

int b2sd_state_set_control_scales(b2sd_handle h, b2sd_state_handle state, const float* per_net_slot, void* stream) {
    return state_set_control_scales("b2sd_state_set_control_scales", h, state, per_net_slot, stream);
}

// n rows of image tokens (nullptr: none) into h->ip_tok, the rest zeroed
static int load_image_tokens(const char* fn, b2sd_handle h, const void* tokens, int n, float scale, cudaStream_t s) {
    if (!h->cfg.ip_tokens) {
        b2_set_error("%s: the engine was created without image prompts (b2sd_config.ip_tokens = 0)", fn);
        return -1;
    }
    if (tokens && (n < 1 || n > h->cfg.ip_tokens || !isfinite(scale))) {
        b2_set_error("%s: n_tok must be 1..%d and scale finite (got %d, %f)", fn, h->cfg.ip_tokens, n, (double)scale);
        return -1;
    }
    const size_t row = (size_t)h->cfg.cross_attention_dim * 2;
    if (!tokens) n = 0;
    if (n) CUDA_OK(cudaMemcpyAsync(h->ip_tok, tokens, n * row, cudaMemcpyDefault, s));
    CUDA_OK(cudaMemsetAsync(reinterpret_cast<char*>(h->ip_tok) + n * row, 0, (ATTN_IP_KEYS - n) * row, s));
    return 0;
}

int b2sd_set_image_embeds(b2sd_handle h, const void* tokens_f16, int n_tok, float scale, void* stream) {
    if (!h || !h->built) {
        b2_set_error("b2sd_set_image_embeds: call b2sd_prepare first");
        return -1;
    }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    TRY(load_image_tokens("b2sd_set_image_embeds", h, tokens_f16, n_tok, scale, s));
    CUDA_OK(cudaStreamSynchronize(s));   // as b2sd_set_prompt_embeds: the caller's host buffer may go once this returns
    h->ip_n_global = tokens_f16 ? n_tok : 0;
    h->ip_scale_global = tokens_f16 ? scale : 1.f;
    CUDA_OK(cudaMemcpyAsync(h->ip_tok_global, h->ip_tok, (size_t)ATTN_IP_KEYS * h->cfg.cross_attention_dim * 2,
                            cudaMemcpyDeviceToDevice, s));
    // the block holds the global text part before the image program overwrites the image part
    TRY(bind_block(h, COND_PROMPT, nullptr, s));
    h->cond[COND_PROMPT].held = COND_UNKNOWN;
    TRY(run_image(h, h->ip_n_global, h->ip_scale_global, s));
    return keep_global(h, COND_PROMPT, s);
}

int b2sd_state_set_image_embeds(b2sd_handle h, b2sd_state_handle state, const void* tokens_f16, int n_tok, float scale,
                                void* stream) {
    const char* fn = "b2sd_state_set_image_embeds";
    TRY(check_state(fn, h, state));
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    TRY(load_image_tokens(fn, h, tokens_f16, n_tok, scale, s));
    CondOverride* base = prompt_base(h, state, true);   // the state's text part: its own prompt's, or the global one
    TRY(bind_block(h, COND_PROMPT, base, s));
    h->cond[COND_PROMPT].held = COND_UNKNOWN;
    const int rc = run_image(h, tokens_f16 ? n_tok : 0, scale, s);
    CUDA_OK(cudaMemcpyAsync(h->ip_tok, h->ip_tok_global, (size_t)ATTN_IP_KEYS * h->cfg.cross_attention_dim * 2,
                            cudaMemcpyDeviceToDevice, s));
    TRY(rc);
    return publish_override(h, state, COND_PROMPT, s, base != nullptr);
}

int b2sd_state_clear_conditioning(b2sd_state_handle state, int which) {
    if (!state || (which != COND_PROMPT && which != COND_TIME)) {
        b2_set_error("b2sd_state_clear_conditioning: null state, or which is not 0 (prompt) or 1 (time)");
        return -1;
    }
    state->cond[which].reset();
    return 0;
}

int64_t b2sd_conditioning_binds(b2sd_handle h) { return h ? h->cond_binds : -1; }

// ---- Canny thresholds: host values, passed to canny_head by the steps submitted after the call -----------------------------
static int check_canny_thresholds(const char* fn, bool canny, double low, double high) {
    if (!canny) {
        b2_set_error("%s: the engine has no ControlNet with the Canny processor", fn);
        return -1;
    }
    if (!isfinite(low) || !isfinite(high)) {
        b2_set_error("%s: the thresholds must be finite (got %f, %f)", fn, low, high);
        return -1;
    }
    return 0;
}

int b2sd_set_canny_thresholds(b2sd_handle h, double low, double high) {
    if (!h) {
        b2_set_error("b2sd_set_canny_thresholds: null handle");
        return -1;
    }
    TRY(check_canny_thresholds("b2sd_set_canny_thresholds", h->reads_canny(), low, high));
    h->canny_low = low;
    h->canny_high = high;
    return 0;
}

int b2sd_state_set_canny_thresholds(b2sd_state_handle state, double low, double high) {
    if (!state) {
        b2_set_error("b2sd_state_set_canny_thresholds: null state");
        return -1;
    }
    TRY(check_canny_thresholds("b2sd_state_set_canny_thresholds", state->canny, low, high));
    state->canny_own = true;
    state->canny_low = low;
    state->canny_high = high;
    return 0;
}

int b2sd_state_clear_canny_thresholds(b2sd_state_handle state) {
    if (!state) {
        b2_set_error("b2sd_state_clear_canny_thresholds: null state");
        return -1;
    }
    TRY(check_canny_thresholds("b2sd_state_clear_canny_thresholds", state->canny, 0, 0));
    state->canny_own = false;
    return 0;
}

int b2sd_step(b2sd_handle h, const void* frame_in, int in_h, int in_w, void* frame_out, void* stream) {
    return b2sd_step_ex(h, frame_in, B2SD_IN_U8_NHWC, in_h, in_w, frame_out, B2SD_OUT_U8_NCHW, stream);
}

// The input heads of a frame, in launch order: the encoder head, and with a ControlNet the head that reads the frame as the
// control image -- the frame itself in [0, 1] at the engine's size (same nearest resize), or HED's edge map, whose first conv
// reads the frame here and whose remaining layers run in stage 1, or Canny's classification of the frame's pixels, whose
// hysteresis runs in stage 1.  With several nets: HED's head and Canny's head once each, before the first net that reads
// their edge map, and one head per net that reads the frame, in net order.
struct InputHead {
    bool canny = false;   // canny_head with `edge`, else smallconv with `conv`
    SmallConvArgs conv{};
    CannyHeadArgs edge{};
    const char* label = nullptr;
    b2sd_launch_record record() const {
        if (!canny) return smallconv_record(conv);
        b2sd_launch_record r{};
        r.kind = B2SD_LAUNCH_CANNY_HEAD;
        r.canny_head = b2sd_canny_head_args{edge.x, edge.in_flags, edge.in_h, edge.in_w, edge.h, edge.w, edge.low, edge.high, edge.cls};
        return r;
    }
    int launch(cudaStream_t s) const { return canny ? canny_head_launch(edge, s) : smallconv_launch(conv, s); }
};
struct InputHeads {
    InputHead head[1 + B2SD_MAX_CONTROLNETS];
    int n = 0;
};

// `state`: the stepped state (its own Canny thresholds, if it has some), or nullptr
static InputHeads input_heads(b2sd_handle h, const b2sd_state* state, const void* frame_in, int in_kind, int in_h, int in_w) {
    const int in_flags = in_kind == B2SD_IN_U8_NHWC ? SC_IN_U8 : (in_kind == B2SD_IN_F32_NCHW ? SC_IN_F32_NCHW : SC_IN_F16_NCHW);
    InputHeads in;
    in.head[0].conv = h->head;
    in.head[0].conv.flags = in_flags | (h->head.flags & SC_IN_OFFSET);   // AutoencoderKL: 2x - 1 as the offset input mode
    in.head[0].label = "smallconv head";
    in.n = 1;
    static const char* cn_label[B2SD_MAX_CONTROLNETS] = {"smallconv controlnet head", "smallconv controlnet1 head",
                                                         "smallconv controlnet2 head", "smallconv controlnet3 head"};
    bool hed_done = false, canny_done = false;
    for (int i = 0; i < h->cfg.controlnet; ++i) {
        const int proc = h->control_processor(i);
        InputHead& e = in.head[in.n];
        if (proc == B2SD_CONTROL_CANNY) {
            if (canny_done) continue;
            canny_done = true;
            const bool own = state && state->canny_own;
            e.canny = true;
            e.edge = CannyHeadArgs{frame_in, in_flags, in_h, in_w, h->cfg.height, h->cfg.width, 0, 0, h->canny_cls};
            canny_thresholds(own ? state->canny_low : h->canny_low, own ? state->canny_high : h->canny_high, &e.edge.low,
                             &e.edge.high);
            e.label = "canny_head";
            ++in.n;
            continue;
        }
        const bool hed = proc == B2SD_CONTROL_HED;
        if (hed && hed_done) continue;
        hed_done = hed_done || hed;
        e.conv = hed ? h->hed_head : h->cn_head[i];
        e.conv.flags = in_flags | (hed ? SC_IN_OFFSET | SC_OUT_RELU : SC_OUT_SILU);
        e.label = hed ? "smallconv hed head" : cn_label[i];
        ++in.n;
    }
    for (int i = 0; i < in.n; ++i) {
        SmallConvArgs& c = in.head[i].conv;
        c.x = frame_in; c.in_h = in_h; c.in_w = in_w;
    }
    return in;
}

static int step_heads(b2sd_handle h, const b2sd_state* state, const void* frame_in, int in_kind, int in_h, int in_w,
                      cudaStream_t s) {
    const InputHeads in = input_heads(h, state, frame_in, in_kind, in_h, in_w);
    for (int i = 0; i < in.n; ++i) TRY(in.head[i].launch(s));
    return 0;
}

// prog_frame[a, b) on s: with use_cuda_graph as the CUDA graph h->graph_exec[slot], captured and instantiated on first use
static int run_frame(b2sd_handle h, int slot, size_t a, size_t b, cudaStream_t s) {
    if (!h->cfg.use_cuda_graph) return h->run(h->prog_frame, s, a, b);
    cudaGraphExec_t& exec = h->graph_exec[slot];
    if (!exec) {
        cudaStream_t cs;   // the caller's stream may be the legacy default stream, which cannot capture
        CUDA_OK(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
        CUDA_OK(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
        const int rc = h->run(h->prog_frame, cs, a, b);
        cudaGraph_t graph = nullptr;
        const cudaError_t ec = cudaStreamEndCapture(cs, &graph);
        cudaStreamDestroy(cs);
        const bool ok = !rc && ec == cudaSuccess && cudaGraphInstantiate(&exec, graph, 0) == cudaSuccess;
        if (graph) cudaGraphDestroy(graph);   // the executable graph does not need it
        if (!ok) {
            exec = nullptr;   // a failed capture must not leave a half-built graph behind
            if (!rc) {
                const char* why = cudaGetErrorString(ec != cudaSuccess ? ec : cudaGetLastError());
                if (slot == b2sd_engine::GRAPH_WHOLE)
                    b2_set_error("b2sd_step: CUDA graph capture / instantiation failed: %s", why);
                else
                    b2_set_error("b2sd_step: CUDA graph capture of stage %d failed: %s", slot - b2sd_engine::GRAPH_STAGE, why);
            }
            return -1;
        }
    }
    CUDA_OK(cudaGraphLaunch(exec, s));
    return 0;
}

// the frame program on a stream state: encoder body | [wait for the state's previous step, state -> slots 1..T-1] last encoder
// conv, UNet, scheduler step [slots 1..T-1 -> state, signal] | decoder.  Only the middle stage is serialised per state: the
// stages of other states, and the other stages of this one, overlap on other lanes.  The copies and the wait stay outside the
// stage graphs because the state changes from frame to frame.
static int step_stages(b2sd_handle h, b2sd_state* state, cudaStream_t s) {
    const size_t cut[4] = {0, h->idx_enc_end, h->idx_unet_end, h->prog_frame.size()};
    __half* slots = h->x_in.p + (size_t)h->lh * h->lw * 4;   // slot 1
    for (int st = 0; st < 3; ++st) {
        if (st == 1) {
            CUDA_OK(cudaStreamWaitEvent(s, state->done, 0));
            if (state->bytes) CUDA_OK(cudaMemcpyAsync(slots, state->buf, state->bytes, cudaMemcpyDeviceToDevice, s));
            TRY(bind_conditioning(h, state, s));
        }
        TRY(run_frame(h, b2sd_engine::GRAPH_STAGE + st, cut[st], cut[st + 1], s));
        if (st == 1) {
            if (state->bytes) CUDA_OK(cudaMemcpyAsync(state->buf, slots, state->bytes, cudaMemcpyDeviceToDevice, s));
            CUDA_OK(cudaEventRecord(state->done, s));
        }
    }
    return 0;
}

static int step_tail(b2sd_handle h, void* frame_out, int out_kind, cudaStream_t s) {
    if (out_kind == B2SD_OUT_F16_NCHW)
        return post_f16_launch(h->image.p, h->image.ld, static_cast<__half*>(frame_out), 1, h->cfg.height, h->cfg.width, s);
    return post_u8_launch(h->image.p, h->image.ld, static_cast<uint8_t*>(frame_out), 1, h->cfg.height, h->cfg.width, s);
}

// b2sd_step_ex with the conditioning of `cond` (nullptr: the engine's global values) bound before the whole-frame program
static int step_whole(b2sd_handle h, const b2sd_state* cond, const void* frame_in, int in_kind, int in_h, int in_w,
                      void* frame_out, int out_kind, void* stream) {
    if (!h || !h->built) {
        b2_set_error("b2sd_step: call b2sd_prepare first");
        return -1;
    }
    if (!frame_in || !frame_out || in_h < 1 || in_w < 1) {
        b2_set_error("b2sd_step: bad frame arguments");
        return -1;
    }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    TRY(step_heads(h, cond, frame_in, in_kind, in_h, in_w, s));
    TRY(bind_conditioning(h, cond, s));
    TRY(run_frame(h, b2sd_engine::GRAPH_WHOLE, 0, h->prog_frame.size(), s));
    return step_tail(h, frame_out, out_kind, s);
}

int b2sd_step_ex(b2sd_handle h, const void* frame_in, int in_kind, int in_h, int in_w, void* frame_out, int out_kind,
                 void* stream) {
    return step_whole(h, nullptr, frame_in, in_kind, in_h, in_w, frame_out, out_kind, stream);
}

int b2sd_state_create(b2sd_handle h, b2sd_state_handle* out, void* stream) {
    if (!h || !out || !h->built) {
        b2_set_error("b2sd_state_create: null argument, or b2sd_prepare not called");
        return -1;
    }
    return state_new(h, reinterpret_cast<cudaStream_t>(stream), out);
}

int b2sd_state_reset(b2sd_state_handle state, void* stream) {
    if (!state) {
        b2_set_error("b2sd_state_reset: null state");
        return -1;
    }
    return state_reset(state, reinterpret_cast<cudaStream_t>(stream));
}

int b2sd_state_destroy(b2sd_state_handle state, void* stream) {
    return state ? state_free(state, reinterpret_cast<cudaStream_t>(stream)) : 0;
}

int b2sd_step_state(b2sd_handle h, b2sd_state_handle state, const void* frame_in, int in_kind, int in_h, int in_w,
                    void* frame_out, int out_kind, void* stream) {
    TRY(check_state("b2sd_step_state", h, state));
    if (!state->bytes) return step_whole(h, state, frame_in, in_kind, in_h, in_w, frame_out, out_kind, stream);
    if (!frame_in || !frame_out || in_h < 1 || in_w < 1) {
        b2_set_error("b2sd_step_state: bad frame arguments");
        return -1;
    }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    TRY(step_heads(h, state, frame_in, in_kind, in_h, in_w, s));
    TRY(step_stages(h, state, s));
    return step_tail(h, frame_out, out_kind, s);
}

int b2sd_get_tensor(b2sd_handle h, const char* name, void* dst, int64_t capacity, int64_t* count, int* dims4, void* stream) {
    if (!h || !h->built || !name) {
        b2_set_error("b2sd_get_tensor: engine not prepared");
        return -1;
    }
    auto u8 = h->u8_taps.find(name);
    if (u8 != h->u8_taps.end()) {
        const b2sd_engine::U8Tap& t = u8->second;
        const int64_t n = (int64_t)t.h * t.w * t.c;
        if (count) *count = n;
        if (dims4) { dims4[0] = 1; dims4[1] = t.h; dims4[2] = t.w; dims4[3] = t.c; }
        if (!dst) return 0;
        if (capacity < n) {
            b2_set_error("b2sd_get_tensor: capacity %lld < %lld", (long long)capacity, (long long)n);
            return -1;
        }
        CUDA_OK(cudaStreamSynchronize(reinterpret_cast<cudaStream_t>(stream)));
        std::vector<uint8_t> host((size_t)n);
        CUDA_OK(cudaMemcpy(host.data(), t.p, (size_t)n, cudaMemcpyDeviceToHost));
        __half* d = static_cast<__half*>(dst);
        for (int64_t i = 0; i < n; ++i) d[i] = __float2half((float)host[i]);   // 0..255: exact in fp16
        return 0;
    }
    auto it = h->taps.find(name);
    if (it == h->taps.end()) {
        b2_set_error("b2sd_get_tensor: unknown tap '%s'", name);
        return -1;
    }
    const Act& a = it->second;
    const int64_t n = (int64_t)a.n * a.h * a.w * a.c;
    if (count) *count = n;
    if (dims4) { dims4[0] = a.n; dims4[1] = a.h; dims4[2] = a.w; dims4[3] = a.c; }
    if (!dst) return 0;
    if (capacity < n) {
        b2_set_error("b2sd_get_tensor: capacity %lld < %lld", (long long)capacity, (long long)n);
        return -1;
    }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    CUDA_OK(cudaStreamSynchronize(s));
    CUDA_OK(cudaMemcpy2D(dst, (size_t)a.c * 2, a.p, (size_t)a.ld * 2, (size_t)a.c * 2, (size_t)a.n * a.h * a.w, cudaMemcpyDeviceToHost));
    return 0;
}

// Eager (non-graph) replay with a CUDA event after every launch: per-op device time, averaged over `iters`.
// Writes a JSON array [{"name": ..., "ms": ...}, ...] into json_buf.  Profiling aid, not the timed path.
int b2sd_profile(b2sd_handle h, const void* frame_in, int in_h, int in_w, void* frame_out, int iters, char* json_buf,
                 int64_t cap, void* stream) {
    if (!h || !h->built || !json_buf || cap < 64) {
        b2_set_error("b2sd_profile: bad arguments");
        return -1;
    }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    TRY(bind_conditioning(h, nullptr, s));
    const size_t nops = h->prog_frame.size() + 2;
    std::vector<cudaEvent_t> ev(nops + 1);
    for (auto& e : ev) CUDA_OK(cudaEventCreate(&e));
    std::vector<double> acc(nops, 0.0);
    for (int it = 0; it < iters + 1; ++it) {  // first iteration is a warm-up
        CUDA_OK(cudaEventRecord(ev[0], s));
        TRY(step_heads(h, nullptr, frame_in, B2SD_IN_U8_NHWC, in_h, in_w, s));
        CUDA_OK(cudaEventRecord(ev[1], s));
        size_t i = 1;
        for (auto& op : h->prog_frame) {
            TRY(op(s));
            ++i;
            CUDA_OK(cudaEventRecord(ev[i], s));
        }
        TRY(post_u8_launch(h->image.p, h->image.ld, static_cast<uint8_t*>(frame_out), 1, h->cfg.height, h->cfg.width, s));
        CUDA_OK(cudaEventRecord(ev[nops], s));
        CUDA_OK(cudaStreamSynchronize(s));
        if (it == 0) continue;
        for (size_t k = 0; k < nops; ++k) {
            float ms = 0.f;
            CUDA_OK(cudaEventElapsedTime(&ms, ev[k], ev[k + 1]));
            acc[k] += ms;
        }
    }
    for (auto& e : ev) cudaEventDestroy(e);
    std::string js = "[";
    char tmp[512];
    for (size_t k = 0; k < nops; ++k) {
        const char* nm = k == 0 ? "smallconv head (u8 frame -> encoder conv_in)" : (k == nops - 1 ? "post_u8 tail" : h->prog_frame[k - 1].name.c_str());
        const double fl = (k == 0 || k == nops - 1) ? 0.0 : h->prog_frame[k - 1].flops;
        snprintf(tmp, sizeof(tmp), "%s{\"name\": \"%s\", \"ms\": %.6f, \"flops\": %.0f}", k ? ", " : "", nm, acc[k] / iters, fl);
        js += tmp;
    }
    js += "]";
    if ((int64_t)js.size() + 1 > cap) {
        b2_set_error("b2sd_profile: buffer too small (%zu needed)", js.size() + 1);
        return -1;
    }
    memcpy(json_buf, js.c_str(), js.size() + 1);
    return 0;
}

// The caller's check around every kernel launch of b2sd_audit_step / b2sd_audit_refresh (see b2sd.h).  Test aid: the stream is
// synchronised twice per launch.
struct Audited {
    const char* entry;
    b2sd_audit_fn fn;
    void* user;
    cudaStream_t s;
    int index = 0;
    int launch(b2sd_launch_record rec, const char* label, const std::function<int()>& run) {
        rec.label = label;
        CUDA_OK(cudaStreamSynchronize(s));
        if (fn(user, index, 0, &rec)) {
            b2_set_error("%s: launch %d '%s' rejected before it ran", entry, index, label);
            return -1;
        }
        TRY(run());
        CUDA_OK(cudaStreamSynchronize(s));
        if (fn(user, index, 1, &rec)) {
            b2_set_error("%s: launch %d '%s' failed its check", entry, index, label);
            return -1;
        }
        ++index;
        return 0;
    }
    int program(std::vector<Op>& ops) {
        for (auto& op : ops) {
            if (op.name.compare(0, 7, "memset ") == 0) {   // a memset node, not a kernel launch
                TRY(op(s));
                continue;
            }
            TRY(launch(op.rec, op.name.c_str(), [&] { return op(s); }));
        }
        return 0;
    }
};

// b2sd_step with the frame program run eagerly
int b2sd_audit_step(b2sd_handle h, const void* frame_in, int in_h, int in_w, void* frame_out, b2sd_audit_fn fn, void* user,
                    void* stream) {
    if (!h || !h->built || !fn || !frame_in || !frame_out || in_h < 1 || in_w < 1) {
        b2_set_error("b2sd_audit_step: bad arguments (or b2sd_prepare not called)");
        return -1;
    }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    TRY(bind_conditioning(h, nullptr, s));   // the engine's own stream: its global conditioning
    Audited au{"b2sd_audit_step", fn, user, s};
    // the input heads and the tail as b2sd_step_ex launches them for a u8 frame, with the caller's frame and size
    const InputHeads in = input_heads(h, nullptr, frame_in, B2SD_IN_U8_NHWC, in_h, in_w);
    for (int i = 0; i < in.n; ++i) {
        const InputHead& e = in.head[i];
        TRY(au.launch(e.record(), e.label, [&] { return e.launch(s); }));
    }
    TRY(au.program(h->prog_frame));
    uint8_t* out = static_cast<uint8_t*>(frame_out);
    TRY(au.launch(post_u8_record(h->image.p, h->image.ld, out, 1, h->cfg.height, h->cfg.width), "post_u8",
                  [&] { return post_u8_launch(h->image.p, h->image.ld, out, 1, h->cfg.height, h->cfg.width, s); }));
    if (au.index != h->launches) {
        b2_set_error("b2sd_audit_step: %d launches audited, %d expected", au.index, h->launches);
        return -1;
    }
    return 0;
}

// b2sd_prepare's refresh (prompt program, then refresh_time) run eagerly
int b2sd_audit_refresh(b2sd_handle h, b2sd_audit_fn fn, void* user, void* stream) {
    if (!h || !h->built || !fn) {
        b2_set_error("b2sd_audit_refresh: bad arguments (or b2sd_prepare not called)");
        return -1;
    }
    Audited au{"b2sd_audit_refresh", fn, user, reinterpret_cast<cudaStream_t>(stream)};
    std::vector<Op> time_ops;
    TRY(time_embedding_ops(h, &time_ops));
    h->cond[COND_PROMPT].held = h->cond[COND_TIME].held = COND_UNKNOWN;
    TRY(write_global_scales(h, au.s));
    TRY(au.program(h->prog_prompt));
    TRY(au.program(time_ops));
    TRY(au.program(h->prog_time));
    h->cond[COND_PROMPT].held = h->cond[COND_TIME].held = COND_GLOBAL;   // recomputed from the global embeddings / timesteps
    return 0;
}

// Start gate for concurrent b2sd_profile_kind calls (one host thread per lane): every call finishes its capture / instantiation /
// warm-up replays, then waits here until all participants have arrived, so that the TIMED replays of the lanes really overlap.
static std::atomic<int> g_gate_expected{0}, g_gate_arrived{0};
int b2sd_profile_gate(int participants) {
    g_gate_arrived.store(0);
    g_gate_expected.store(participants > 1 ? participants : 0);
    return 0;
}

// Device time of one launch class inside a CUDA graph: every frame-program launch whose label starts with `kind`
// ("igemm", "attn", "groupnorm", ...) is captured, in program order, into its own graph (same PDL edges, same buffers,
// same weight streaming as the frame graph) and that graph is replayed `iters` times between two events.
int b2sd_profile_kind(b2sd_handle h, const char* kind, int iters, double* ms_per_replay, int* launches, double* flops,
                      void* stream) {
    if (!h || !h->built || !kind || iters < 1 || !ms_per_replay) {
        b2_set_error("b2sd_profile_kind: bad arguments");
        return -1;
    }
    cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
    const std::string k(kind);
    int n = 0;
    double fl = 0.0;
    for (auto& op : h->prog_frame)   // eager pass first: one-time attribute/driver-entry-point setup may not run under capture
        if (op.name.compare(0, k.size(), k) == 0) { TRY(op(s)); ++n; fl += op.flops; }
    CUDA_OK(cudaStreamSynchronize(s));
    if (n == 0) {
        b2_set_error("b2sd_profile_kind: no launch of kind '%s'", kind);
        return -1;
    }
    cudaGraph_t g = nullptr;
    cudaGraphExec_t ge = nullptr;
    cudaStream_t cs;   // the caller's stream may be the legacy default stream, which cannot capture
    CUDA_OK(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
    CUDA_OK(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
    int rc = 0;
    for (auto& op : h->prog_frame)
        if (op.name.compare(0, k.size(), k) == 0 && op(cs)) { rc = -1; break; }
    cudaError_t ce = cudaStreamEndCapture(cs, &g);
    cudaStreamDestroy(cs);
    if (rc || ce != cudaSuccess) {
        if (g) cudaGraphDestroy(g);
        if (!rc) b2_set_error("b2sd_profile_kind: capture failed: %s", cudaGetErrorString(ce));
        return -1;
    }
    CUDA_OK(cudaGraphInstantiate(&ge, g, 0));
    cudaEvent_t e0, e1;
    CUDA_OK(cudaEventCreate(&e0));
    CUDA_OK(cudaEventCreate(&e1));
    for (int i = 0; i < 3; ++i) CUDA_OK(cudaGraphLaunch(ge, s));
    CUDA_OK(cudaStreamSynchronize(s));
    if (const int expect = g_gate_expected.load()) {   // concurrent measurement: start the timed replays together
        g_gate_arrived.fetch_add(1);
        const auto t0 = std::chrono::steady_clock::now();
        while (g_gate_arrived.load() < expect && std::chrono::steady_clock::now() - t0 < std::chrono::seconds(20))
            std::this_thread::sleep_for(std::chrono::microseconds(50));
    }
    CUDA_OK(cudaEventRecord(e0, s));
    for (int i = 0; i < iters; ++i) CUDA_OK(cudaGraphLaunch(ge, s));
    CUDA_OK(cudaEventRecord(e1, s));
    CUDA_OK(cudaStreamSynchronize(s));
    float ms = 0.f;
    CUDA_OK(cudaEventElapsedTime(&ms, e0, e1));
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaGraphExecDestroy(ge);
    cudaGraphDestroy(g);
    *ms_per_replay = (double)ms / iters;
    if (launches) *launches = n;
    if (flops) *flops = fl;
    return 0;
}

int b2sd_launches_per_step(b2sd_handle h) { return h ? h->launches : 0; }

int b2sd_set_concurrency(b2sd_handle h, int frames_in_flight) {
    if (!h || frames_in_flight < 1) {
        b2_set_error("b2sd_set_concurrency: bad argument");
        return -1;
    }
    h->concurrency = frames_in_flight;
    h->built = false;   // the launch policy is applied when the frame program is built (b2sd_prepare)
    return 0;
}

}  // extern "C"
