// Band-limited sinc resampling (torchaudio.functional.resample, method "sinc_interp_hann", lowpass_filter_width = 6,
// rolloff = 0.99) for offline batches (fac_resample) and live sessions (fac_rs_pool_*).
//
// With the rates reduced by their gcd to (orig, new): base = min(orig, new) * 0.99, width = ceil(6 orig / base),
// K = 2 width + orig taps per phase and `new` phases.  Lane input x[0, n) gives ceil(new n / orig) outputs; output j has
// block i = j / new and phase p = j % new and is
//
//     y[j] = sum over k = 0 .. K-1 of h[p][k] * x[i orig - width + k],      x[m] = 0 outside [0, n)
//
// summed in fp32 as acc = fmaf(h[p][k], x[.], acc), k ascending from acc = 0.  ONE thread computes one output over its
// whole window, and the order depends on nothing but (p, k): not on where j falls in a tile, a launch, a lane batch or a
// stream chunk.  That is what makes a ragged lane equal its own B = 1 call and a stream equal its offline call, bit for
// bit.  The table h [new][K] is the float32 one torchaudio builds for float32 input; the caller registers it per pair
// (fac_resample_table).  Equal rates reduce to (1, 1) with the one-tap table {1}: a copy.
//
// Launch: one CTA per (output tile, lane).  Each lane brings its own pair, table, outputs and input, which is the logical
// concatenation of two spans (a stream's history and its new chunk; an offline lane has only the second).  A CTA stages
// its tile's input window (tile span + K samples) in shared memory with coalesced loads, and the table too when it holds at
// most kRsSmemTable floats; larger tables are read through __ldg.  The device keeps h transposed, [K][new], so the threads
// of a warp (consecutive phases) read consecutive words of it at every k.  A stream step's CTAs also copy the lane's new history
// to the session's other buffer (double buffering: the host flips the slot only after the launch is queued).
#include <algorithm>
#include <climits>
#include <cmath>
#include <map>
#include <memory>
#include <utility>
#include <vector>

#include "../../include/facodec_b200.h"
#include "resample.h"

namespace fac {

namespace {

constexpr int kRsTile = 256;          // outputs (threads) per CTA
constexpr int kRsLanes = 256;         // lanes per launch: the lane table is a kernel parameter (<= 32 KB on sm_90)
constexpr int kRsSmemTable = 4096;    // tables of at most this many floats are staged in shared memory
constexpr int kRsMaxTable = 65536;    // K * new of a supported pair
constexpr int kRsRateMin = 8000, kRsRateMax = 192000;

struct RsLane {
    const float* tab;     // h transposed, [K][new]: a warp's consecutive phases read consecutive words
    const float* a;       // logical input [s0, s0 + la)
    const float* b;       // logical input [s0 + la, s0 + la + lb)
    float* y;             // outputs j0 .. j0 + n_write - 1 (zeros from n_out on)
    float* hist;          // receives logical [s0 + h0, s0 + h0 + hl), or null
    long long s0, j0, n;  // first logical index of a, first output, input length (x[m] = 0 for m >= n)
    int la, lb, n_out, n_write, h0, hl;
    int orig, nw, width, K, tab_smem;
};
struct RsParams {
    RsLane lane[kRsLanes];
};

__global__ void __launch_bounds__(kRsTile) resample_kernel(const __grid_constant__ RsParams p) {
    const RsLane& L = p.lane[blockIdx.y];
    extern __shared__ float sm[];
    const int tid = threadIdx.x;
    for (int q = blockIdx.x * kRsTile + tid; q < L.hl; q += gridDim.x * kRsTile) {
        const int m = L.h0 + q;
        L.hist[q] = m < L.la ? L.a[m] : L.b[m - L.la];
    }
    const long long jt = (long long)blockIdx.x * kRsTile;
    if (jt >= L.n_write) return;                                  // uniform over the CTA
    const int j = (int)jt + tid;
    if (jt < L.n_out) {                                           // uniform over the CTA
        const long long g0 = L.j0 + jt;
        const long long i0 = g0 / L.nw;                           // block of the tile's first output
        const int r0 = (int)(g0 - i0 * L.nw);                     // its phase
        const int last = (int)((jt + kRsTile < L.n_out ? jt + kRsTile : (long long)L.n_out) - 1 - jt);
        const long long lo = i0 * L.orig - L.width;               // logical index of xs[0]
        const int span = (r0 + last) / L.nw * L.orig + L.K;
        const int tabn = L.tab_smem ? L.nw * L.K : 0;
        float* ts = sm;
        float* xs = sm + tabn;
        for (int q = tid; q < tabn; q += kRsTile) ts[q] = __ldg(L.tab + q);
        for (int q = tid; q < span; q += kRsTile) {
            const long long m = lo + q;
            float v = 0.f;
            if (m >= 0 && m < L.n) {
                const long long r = m - L.s0;
                v = r < L.la ? __ldg(L.a + r) : __ldg(L.b + (r - L.la));
            }
            xs[q] = v;
        }
        __syncthreads();
        if (j < L.n_out) {
            const int di = (r0 + tid) / L.nw;                     // block and phase of output j, relative to the tile
            const int ph = r0 + tid - di * L.nw;
            const float* xw = xs + di * L.orig;
            float acc = 0.f;
            if (L.tab_smem) {
                for (int k = 0; k < L.K; ++k) acc = fmaf(ts[k * L.nw + ph], xw[k], acc);
            } else {
                for (int k = 0; k < L.K; ++k) acc = fmaf(__ldg(L.tab + (size_t)k * L.nw + ph), xw[k], acc);
            }
            L.y[j] = acc;
            return;
        }
    }
    if (j < L.n_write) L.y[j] = 0.f;
}

long long gcd_ll(long long a, long long b) { while (b) { long long t = a % b; a = b; b = t; } return a; }

struct RsTable { int orig = 0, nw = 0, width = 0, K = 0; float* dev = nullptr; };

struct RsSlot {
    bool used = false, finished = false;
    int orig = 0, nw = 0, width = 0, K = 0;
    const float* tab = nullptr;
    long long seen = 0, emitted = 0, hs = 0;   // samples pushed, outputs returned, logical index of the history's first sample
    int hl = 0, cur = 0, cap = 0;              // history length, current buffer, capacity of each buffer (floats)
    float* buf[2] = {nullptr, nullptr};
};

struct RsPool {
    int quantum = 1;
    std::vector<RsSlot> slot;
    std::vector<RsSlot> prev;         // each slot before its last step, while that step can be taken back (undo[i])
    std::vector<char> undo;
};

// Worst-case history of a slot: the input from the window of the first output not yet returned.  Without a quantum that
// is < K samples; a quantum q holds back up to q - 1 outputs, ceil((q - 1) / new) blocks of orig samples more.
int hist_cap(int orig, int nw, int K, int q) { return K + orig * ((q - 1 + nw - 1) / nw); }

}  // namespace

struct RsHost {
    std::map<std::pair<int, int>, RsTable> tables;   // by reduced pair
    std::vector<std::unique_ptr<RsPool>> pools;      // a destroyed pool leaves a null entry
    ~RsHost() {
        for (auto& kv : tables) cudaFree(kv.second.dev);
        for (auto& P : pools)
            if (P) for (auto& s : P->slot) { cudaFree(s.buf[0]); cudaFree(s.buf[1]); }
    }
};

int rs_geometry(int orig, int nw, int* out4) {
    if (orig < kRsRateMin || orig > kRsRateMax || nw < kRsRateMin || nw > kRsRateMax) return FAC_ERR_INVALID;
    const long long g = gcd_ll(orig, nw);
    const int o = (int)(orig / g), n = (int)(nw / g);
    int width = 0, K = 1;
    if (o != n) {
        const double base = (double)std::min(o, n) * 0.99;
        width = (int)std::ceil(6.0 * o / base);
        K = 2 * width + o;
    }
    if ((long long)K * n > kRsMaxTable) return FAC_ERR_INVALID;
    if (out4) { out4[0] = o; out4[1] = n; out4[2] = width; out4[3] = K; }
    return FAC_OK;
}

namespace {
// The counts of a reduced pair (o, n) with its width.
long long out_len_reduced(int o, int n, long long len) { return ((long long)n * len + o - 1) / o; }

long long ready_reduced(int o, int n, int width, int quantum, long long seen, long long emitted) {
    const long long avail = seen < width + o ? 0 : ((seen - width - o) / o + 1) * n;
    return avail <= emitted ? 0 : (avail - emitted) / quantum * quantum;
}
}  // namespace

long long rs_out_len(int orig, int nw, long long n) {
    int g[4];
    if (rs_geometry(orig, nw, g) || n < 0) return FAC_ERR_INVALID;
    return out_len_reduced(g[0], g[1], n);
}

// Outputs a push returns once `seen` samples are in and `emitted` outputs were returned before: those whose whole window
// lies inside the input so far, rounded down to a multiple of the quantum.
long long rs_ready(int orig, int nw, int quantum, long long seen, long long emitted) {
    int g[4];
    if (rs_geometry(orig, nw, g) || quantum < 1 || seen < 0 || emitted < 0) return FAC_ERR_INVALID;
    return ready_reduced(g[0], g[1], g[2], quantum, seen, emitted);
}

namespace {

RsHost& host_of(RsEnv& e) {
    if (!e.host) e.host = new RsHost();
    return *e.host;
}

int unsupported(RsEnv& e, const char* who, int orig, int nw) {
    e.err = std::string(who) + ": unsupported rate pair " + std::to_string(orig) + " -> " + std::to_string(nw) +
            " (integer rates in [8000, 192000] whose reduced table holds at most 65536 floats)";
    return FAC_ERR_INVALID;
}

// The registered table of a pair (the one-tap copy table of equal rates is made here).
int find_table(RsEnv& e, const char* who, int orig, int nw, const RsTable** out) {
    int g[4];
    if (rs_geometry(orig, nw, g)) return unsupported(e, who, orig, nw);
    RsHost& H = host_of(e);
    auto it = H.tables.find({g[0], g[1]});
    if (it == H.tables.end() && g[0] == g[1]) {
        const float one = 1.f;
        int rc = rs_table(e, orig, nw, &one);
        if (rc) return rc;
        it = H.tables.find({g[0], g[1]});
    }
    if (it == H.tables.end()) {
        e.err = std::string(who) + ": no filter table for " + std::to_string(orig) + " -> " + std::to_string(nw) +
                " (register it with fac_resample_table)";
        return FAC_ERR_STATE;
    }
    *out = &it->second;
    return FAC_OK;
}

int smem_bytes(const RsLane& L) {
    const int span = ((kRsTile - 1) / L.nw + 1) * L.orig + L.K;
    return (int)sizeof(float) * (span + (L.tab_smem ? L.nw * L.K : 0));
}

// Launches the lanes, kRsLanes per launch.
int launch_lanes(RsEnv& e, const char* who, std::vector<RsLane>& lanes, cudaStream_t st) {
    cudaError_t err = cudaSetDevice(e.device);
    e.launches = 0;
    for (size_t o = 0; err == cudaSuccess && o < lanes.size(); o += kRsLanes) {
        const int nl = (int)std::min(lanes.size() - o, (size_t)kRsLanes);
        auto P = std::make_unique<RsParams>();
        long long tiles = 1;
        int smem = 0;
        for (int i = 0; i < nl; ++i) {
            RsLane& L = lanes[o + i];
            L.tab_smem = L.nw * L.K <= kRsSmemTable;
            P->lane[i] = L;
            tiles = std::max(tiles, ((long long)L.n_write + kRsTile - 1) / kRsTile);
            smem = std::max(smem, smem_bytes(L));
        }
        if (smem > 48 * 1024) err = cudaFuncSetAttribute(resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        if (err != cudaSuccess) break;
        resample_kernel<<<dim3((unsigned)tiles, (unsigned)nl), kRsTile, smem, st>>>(*P);
        err = cudaGetLastError();
        ++e.launches;
    }
    if (err != cudaSuccess) {
        e.err = std::string(who) + ": " + cudaGetErrorString(err);
        cudaGetLastError();
        return FAC_ERR_CUDA;
    }
    return FAC_OK;
}

RsLane lane_of(const RsTable& t) {
    RsLane L{};
    L.tab = t.dev;
    L.orig = t.orig; L.nw = t.nw; L.width = t.width; L.K = t.K;
    return L;
}

RsLane lane_of(const RsSlot& s) {
    RsLane L{};
    L.tab = s.tab;
    L.orig = s.orig; L.nw = s.nw; L.width = s.width; L.K = s.K;
    return L;
}

}  // namespace

int rs_table(RsEnv e, int orig, int nw, const float* table_host) {
    int g[4];
    if (rs_geometry(orig, nw, g)) return unsupported(e, "fac_resample_table", orig, nw);
    if (!table_host) { e.err = "fac_resample_table: null table"; return FAC_ERR_INVALID; }
    RsHost& H = host_of(e);
    if (H.tables.count({g[0], g[1]})) return FAC_OK;       // one upload per pair and handle
    const int nw_r = g[1], K = g[3];
    const size_t n = (size_t)nw_r * K;
    std::vector<float> tr(n);                               // [new][K] -> [K][new]
    for (int p = 0; p < nw_r; ++p)
        for (int k = 0; k < K; ++k) tr[(size_t)k * nw_r + p] = table_host[(size_t)p * K + k];
    float* d = nullptr;
    cudaError_t err = cudaSetDevice(e.device);
    if (err == cudaSuccess) err = cudaMalloc(&d, n * sizeof(float));
    if (err == cudaSuccess) err = cudaMemcpy(d, tr.data(), n * sizeof(float), cudaMemcpyHostToDevice);
    if (err != cudaSuccess) {
        cudaFree(d);
        e.err = std::string("fac_resample_table: ") + cudaGetErrorString(err);
        cudaGetLastError();
        return FAC_ERR_CUDA;
    }
    H.tables[{g[0], g[1]}] = RsTable{g[0], g[1], g[2], g[3], d};
    return FAC_OK;
}

int rs_resample(RsEnv e, const float* x, int B, int T, const int* lengths, int orig, int nw, float* y, cudaStream_t st) {
    const char* who = "fac_resample";
    if (!x || !y || B < 1 || T < 1) { e.err = "fac_resample: bad arguments (x, y, B >= 1, T >= 1)"; return FAC_ERR_INVALID; }
    const RsTable* t = nullptr;
    int rc = find_table(e, who, orig, nw, &t);
    if (rc) return rc;
    const long long Tout = rs_out_len(orig, nw, T);
    if (Tout > INT_MAX / 2) { e.err = "fac_resample: output too long"; return FAC_ERR_INVALID; }
    std::vector<RsLane> lanes(B);
    for (int b = 0; b < B; ++b) {
        const int n = lengths ? lengths[b] : T;
        if (n < 0 || n > T) {
            e.err = "fac_resample: lengths[" + std::to_string(b) + "] = " + std::to_string(n) + " lies outside [0, " +
                    std::to_string(T) + "]";
            return FAC_ERR_INVALID;
        }
        RsLane& L = lanes[b] = lane_of(*t);
        L.a = x + (size_t)b * T; L.la = n; L.b = nullptr; L.lb = 0;
        L.s0 = 0; L.j0 = 0; L.n = n;
        L.y = y + (size_t)b * Tout;
        L.n_out = (int)rs_out_len(orig, nw, n);
        L.n_write = (int)Tout;
    }
    return launch_lanes(e, who, lanes, st);
}

int rs_pool_create(RsEnv e, int capacity, int quantum) {
    if (capacity < 1 || quantum < 1) { e.err = "fac_rs_pool_create: bad arguments (capacity >= 1, quantum >= 1)"; return FAC_ERR_INVALID; }
    RsHost& H = host_of(e);
    auto P = std::make_unique<RsPool>();
    P->quantum = quantum;
    P->slot.resize(capacity);
    P->prev.resize(capacity);
    P->undo.assign(capacity, 0);
    H.pools.push_back(std::move(P));
    return (int)H.pools.size() - 1;
}

namespace {
// Grow-only history buffers of a free slot: a reopened slot keeps its buffers.
int grow_slot(RsEnv& e, RsSlot& s, int cap, const char* who) {
    if (cap <= s.cap) return FAC_OK;
    cudaError_t err = cudaSetDevice(e.device);
    float* b[2] = {nullptr, nullptr};
    for (int k = 0; k < 2 && err == cudaSuccess; ++k) err = cudaMalloc(&b[k], sizeof(float) * cap);
    if (err != cudaSuccess) {
        cudaFree(b[0]); cudaFree(b[1]);
        e.err = std::string(who) + ": " + cudaGetErrorString(err);
        cudaGetLastError();
        return FAC_ERR_CUDA;
    }
    cudaDeviceSynchronize();                         // the old buffers may still be read by queued steps
    cudaFree(s.buf[0]); cudaFree(s.buf[1]);
    s.buf[0] = b[0]; s.buf[1] = b[1]; s.cap = cap;
    return FAC_OK;
}

RsPool* pool_of(RsEnv& e, int id, const char* who) {
    RsHost& H = host_of(e);
    RsPool* P = id >= 0 && id < (int)H.pools.size() ? H.pools[id].get() : nullptr;
    if (!P) e.err = std::string(who) + ": no such pool";
    return P;
}
}  // namespace

int rs_pool_open(RsEnv e, int pool_id, int orig, int nw) {
    const char* who = "fac_rs_pool_open";
    RsPool* P = pool_of(e, pool_id, who);
    if (!P) return FAC_ERR_INVALID;
    const RsTable* t = nullptr;
    int rc = find_table(e, who, orig, nw, &t);
    if (rc) return rc;
    int i = 0;
    while (i < (int)P->slot.size() && P->slot[i].used) ++i;
    if (i == (int)P->slot.size()) {
        e.err = std::string(who) + ": the pool is full (capacity " + std::to_string(P->slot.size()) + ")";
        return FAC_ERR_STATE;
    }
    RsSlot& s = P->slot[i];
    if ((rc = grow_slot(e, s, hist_cap(t->orig, t->nw, t->K, P->quantum), who))) return rc;
    s.used = true; s.finished = false;
    s.orig = t->orig; s.nw = t->nw; s.width = t->width; s.K = t->K; s.tab = t->dev;
    s.seen = s.emitted = s.hs = 0; s.hl = 0; s.cur = 0;
    P->undo[i] = 0;
    return i;
}

int rs_pool_step(RsEnv e, int pool_id, int n, const int* sessions, const int* T, const float* const* x, float* const* y,
                 int* counts, bool finish, cudaStream_t st) {
    const char* who = finish ? "fac_rs_pool_finish" : "fac_rs_pool_push";
    RsPool* P = pool_of(e, pool_id, who);
    if (!P) return FAC_ERR_INVALID;
    if (n < 0 || (n > 0 && (!sessions || !y || !counts || (!finish && (!T || !x))))) {
        e.err = std::string(who) + ": bad arguments";
        return FAC_ERR_INVALID;
    }
    std::vector<char> seen(P->slot.size(), 0);
    std::vector<RsLane> lanes;
    std::vector<RsSlot> next(n);
    for (int i = 0; i < n; ++i) {
        const int sid = sessions[i];
        if (sid < 0 || sid >= (int)P->slot.size() || !P->slot[sid].used || seen[sid]++) {
            e.err = std::string(who) + ": session " + std::to_string(sid) + " is not open or is named twice";
            return FAC_ERR_INVALID;
        }
        const RsSlot& s = P->slot[sid];
        if (s.finished) { e.err = std::string(who) + ": session " + std::to_string(sid) + " is finished"; return FAC_ERR_STATE; }
        const int Ti = T ? T[i] : 0;
        const float* xi = x ? x[i] : nullptr;
        if (Ti < 0 || (Ti > 0 && !xi)) {
            e.err = std::string(who) + ": session " + std::to_string(sid) + ": bad chunk (T >= 0, a buffer when T > 0)";
            return FAC_ERR_INVALID;
        }
        RsSlot& t = next[i] = s;
        t.seen = s.seen + Ti;
        const long long total = finish ? out_len_reduced(s.orig, s.nw, t.seen) - s.emitted
                                       : ready_reduced(s.orig, s.nw, s.width, P->quantum, t.seen, s.emitted);
        if (total > INT_MAX / 2) { e.err = std::string(who) + ": chunk too long"; return FAC_ERR_INVALID; }
        if (total > 0 && !y[i]) { e.err = std::string(who) + ": null output buffer"; return FAC_ERR_INVALID; }
        t.emitted = s.emitted + total;
        RsLane L = lane_of(s);
        L.a = s.buf[s.cur]; L.la = s.hl; L.b = xi; L.lb = Ti;
        L.s0 = s.hs; L.j0 = s.emitted; L.n = t.seen;
        L.y = y[i]; L.n_out = L.n_write = (int)total;
        if (finish) {
            t.finished = true;
            t.hl = 0;
        } else {
            t.hs = std::max(0LL, (t.emitted / s.nw) * s.orig - s.width);
            t.hl = (int)(t.seen - t.hs);
            if (t.hl > s.cap) { e.err = std::string(who) + ": history overflow"; return FAC_ERR_STATE; }
            t.cur = s.cur ^ 1;
            L.hist = s.buf[t.cur]; L.h0 = (int)(t.hs - s.hs); L.hl = t.hl;
        }
        counts[i] = (int)total;
        if (L.n_write > 0 || L.hl > 0) lanes.push_back(L);
    }
    int rc = lanes.empty() ? (e.launches = 0, FAC_OK) : launch_lanes(e, who, lanes, st);
    if (rc) return rc;
    for (int i = 0; i < n; ++i) {                                 // every lane queued: flip the slots
        const int sid = sessions[i];
        P->prev[sid] = P->slot[sid];
        P->undo[sid] = 1;
        P->slot[sid] = next[i];
    }
    return FAC_OK;
}

// The step wrote only the buffer a slot was not reading, so restoring the slot's counters and buffer index takes it back.
int rs_pool_undo(RsEnv e, int pool_id, int n, const int* sessions) {
    const char* who = "fac_rs_pool_undo";
    RsPool* P = pool_of(e, pool_id, who);
    if (!P) return FAC_ERR_INVALID;
    if (n < 0 || (n > 0 && !sessions)) { e.err = std::string(who) + ": bad arguments"; return FAC_ERR_INVALID; }
    std::vector<char> named(P->slot.size(), 0);
    for (int i = 0; i < n; ++i) {
        const int sid = sessions[i];
        if (sid < 0 || sid >= (int)P->slot.size() || !P->slot[sid].used || !P->undo[sid] || named[sid]++) {
            e.err = std::string(who) + ": session " + std::to_string(sid) + " has no step to take back, or is named twice";
            return FAC_ERR_INVALID;
        }
    }
    for (int i = 0; i < n; ++i) {
        P->slot[sessions[i]] = P->prev[sessions[i]];
        P->undo[sessions[i]] = 0;
    }
    return FAC_OK;
}

int rs_pool_close(RsEnv e, int pool_id, int session) {
    RsPool* P = pool_of(e, pool_id, "fac_rs_pool_close");
    if (!P) return FAC_ERR_INVALID;
    if (session < 0 || session >= (int)P->slot.size() || !P->slot[session].used) {
        e.err = "fac_rs_pool_close: session " + std::to_string(session) + " is not open";
        return FAC_ERR_INVALID;
    }
    P->slot[session].used = false;
    P->undo[session] = 0;
    return FAC_OK;
}

int rs_pool_destroy(RsEnv e, int pool_id) {
    RsPool* P = pool_of(e, pool_id, "fac_rs_pool_destroy");
    if (!P) return FAC_ERR_INVALID;
    cudaSetDevice(e.device);
    cudaDeviceSynchronize();
    for (auto& s : P->slot) { cudaFree(s.buf[0]); cudaFree(s.buf[1]); }
    e.host->pools[pool_id].reset();
    return FAC_OK;
}

void rs_host_free(RsHost* host) { delete host; }

// counters: {quantum, orig, new, width, K, seen, emitted, hs, hl} (include/facodec_b200.h, FAC_STATE_RS)
int rs_slot_read(RsEnv e, int pool_id, int session, SlotState& st, const char* who) {
    RsPool* P = pool_of(e, pool_id, who);
    if (!P) return FAC_ERR_INVALID;
    if (session < 0 || session >= (int)P->slot.size() || !P->slot[session].used) {
        e.err = std::string(who) + ": session " + std::to_string(session) + " is not open";
        return FAC_ERR_INVALID;
    }
    const RsSlot& s = P->slot[session];
    if (s.finished) { e.err = std::string(who) + ": session " + std::to_string(session) + " is finished"; return FAC_ERR_STATE; }
    const long long c[9] = {P->quantum, s.orig, s.nw, s.width, s.K, s.seen, s.emitted, s.hs, s.hl};
    std::copy(c, c + 9, st.counters);
    st.nreg = 1;
    st.region[0] = s.buf[s.cur];
    st.bytes[0] = (long long)sizeof(float) * s.hl;
    return FAC_OK;
}

int rs_slot_place(RsEnv e, int pool_id, SlotState& st, const char* who) {
    RsPool* P = pool_of(e, pool_id, who);
    if (!P) return FAC_ERR_INVALID;
    const long long* c = st.counters;
    if (c[0] != P->quantum) {
        e.err = std::string(who) + ": the state's quantum " + std::to_string(c[0]) + " is not the pool's " + std::to_string(P->quantum);
        return FAC_ERR_STATE;
    }
    RsHost& H = host_of(e);
    auto it = H.tables.find({(int)c[1], (int)c[2]});
    if (it == H.tables.end() && c[1] == 1 && c[2] == 1) {               // equal rates: the one-tap copy table
        const float one = 1.f;
        if (int rc = rs_table(e, 24000, 24000, &one)) return rc;
        it = H.tables.find({1, 1});
    }
    if (it == H.tables.end()) {
        e.err = std::string(who) + ": no filter table for the reduced pair " + std::to_string(c[1]) + " -> " + std::to_string(c[2]) +
                " (register it with fac_resample_table)";
        return FAC_ERR_STATE;
    }
    const RsTable& t = it->second;
    const int cap = hist_cap(t.orig, t.nw, t.K, P->quantum);
    const long long seen = c[5], emitted = c[6], hs = c[7], hl = c[8];
    if (c[3] != t.width || c[4] != t.K || seen < 0 || emitted < 0 || emitted > out_len_reduced(t.orig, t.nw, seen) || hs < 0 ||
        hl < 0 || hl > cap || hs + hl != seen || st.bytes[0] != (long long)sizeof(float) * hl ||
        std::any_of(st.bytes + 1, st.bytes + FAC_STATE_REGIONS, [](long long b) { return b != 0; })) {
        e.err = std::string(who) + ": the resampler counters are inconsistent";
        return FAC_ERR_INVALID;
    }
    int i = 0;
    while (i < (int)P->slot.size() && P->slot[i].used) ++i;
    if (i == (int)P->slot.size()) {
        e.err = std::string(who) + ": the pool is full (capacity " + std::to_string(P->slot.size()) + ")";
        return FAC_ERR_STATE;
    }
    RsSlot& s = P->slot[i];
    if (int rc = grow_slot(e, s, cap, who)) return rc;
    s.orig = t.orig; s.nw = t.nw; s.width = t.width; s.K = t.K; s.tab = t.dev;
    st.region[0] = s.buf[0];
    st.nreg = 1;
    return i;
}

void rs_slot_commit(RsEnv e, int pool_id, int slot, const SlotState& st) {
    RsPool* P = pool_of(e, pool_id, "fac_rs_pool_import");
    RsSlot& s = P->slot[slot];
    s.used = true; s.finished = false;
    s.seen = st.counters[5]; s.emitted = st.counters[6]; s.hs = st.counters[7]; s.hl = (int)st.counters[8]; s.cur = 0;
    P->undo[slot] = 0;
}

}  // namespace fac
