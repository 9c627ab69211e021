// Library-wide state and the small utility entry points of the C ABI.
#include "common.cuh"
#include <cstring>
#include "../../include/nunif_b200.h"

#include <mutex>
#include <vector>
#include <map>

namespace nb200 {
thread_local std::string g_last_error;
std::atomic<uint64_t> g_launches{0};
std::atomic<int> g_prof_enabled{0};

struct ProfRec { cudaEvent_t a, b; int cat; double work, rb, wb; };
// HBM rates the per-launch floors are computed with (copy, write-only, read-only, bytes/s): the H100 SXM data-sheet HBM3
// bandwidth, not a measured ceiling
static double g_bw_copy = 3.35e12, g_bw_write = 3.35e12, g_bw_read = 3.35e12;
static std::mutex g_prof_mu;
static std::vector<ProfRec> g_prof_recs;
static std::vector<cudaEvent_t> g_prof_pool;
static const char* kCatNames[PC_COUNT] = {"gemm", "window_attention", "stem_conv", "to_image", "tile_unfold", "tile_blend",
                                          "se_block", "tail_conv", "forward_warp", "backward_warp", "dilate_edge",
                                          "minmax_map", "other", "fused_mlp", "fused_attn", "hole_mask"};

static cudaEvent_t prof_event() {
    if (!g_prof_pool.empty()) { cudaEvent_t e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
    cudaEvent_t e;
    cudaEventCreate(&e);
    return e;
}
void prof_begin(cudaStream_t st, int cat, double work, double rb, double wb) {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    ProfRec r; r.a = prof_event(); r.b = prof_event(); r.cat = cat; r.work = work; r.rb = rb; r.wb = wb;
    cudaEventRecord(r.a, st);
    g_prof_recs.push_back(r);
}
void prof_end(cudaStream_t st) {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    if (!g_prof_recs.empty()) cudaEventRecord(g_prof_recs.back().b, st);
}

std::atomic<int> g_rec_enabled{0};
static std::mutex g_rec_mu;
static std::string g_rec;
RecField::RecField(const char* n, double v) : name(n) {
    char s[32];
    snprintf(s, sizeof(s), "%.9g", v);
    value = s;
}
void rec_launch(const char* kind, std::initializer_list<RecField> fields) {
    std::string line = kind;
    for (const RecField& f : fields) {
        line += ',';
        line += f.name;
        line += '=';
        line += f.value;
    }
    line += '\n';
    std::lock_guard<std::mutex> lk(g_rec_mu);
    g_rec += line;
}

static std::mutex g_attr_mu;
static std::map<std::pair<int, const void*>, size_t> g_dyn_smem;
static std::map<std::pair<int, const void*>, int> g_carveout;
int ensure_dyn_smem(const void* func, size_t bytes, int carveout) {
    int dev = 0;
    NB_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lk(g_attr_mu);
    size_t& have = g_dyn_smem[{dev, func}];
    if (bytes > have && bytes > 48 * 1024) {
        NB_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        have = bytes;
    }
    if (carveout > 0) {
        int& set = g_carveout[{dev, func}];
        if (set != carveout) {
            NB_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributePreferredSharedMemoryCarveout, carveout));
            set = carveout;
        }
    }
    return 0;
}
int ensure_dyn_smem(const void* func, size_t bytes) { return ensure_dyn_smem(func, bytes, 0); }
int device_sm_count() {
    static std::atomic<int> cache[64];
    int dev = 0;
    cudaGetDevice(&dev);
    if (dev < 0 || dev >= 64) dev = 0;
    int n = cache[dev].load(std::memory_order_relaxed);
    if (n <= 0) {
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
        if (n <= 0) n = 148;
        cache[dev].store(n, std::memory_order_relaxed);
    }
    return n;
}
}  // namespace nb200

using namespace nb200;

extern "C" const char* nb200_last_error(void) { return g_last_error.c_str(); }
extern "C" int nb200_abi_version(void) { return NB200_ABI_VERSION; }
extern "C" uint64_t nb200_launch_count(void) { return g_launches.load(); }

extern "C" int nb200_check_device(int device) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return fail("no CUDA device: the nunif_b200 hot path has no CPU fallback");
    NB_CHECK(device >= 0 && device < n, "device index out of range");
    cudaDeviceProp prop;
    NB_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0)   // sm_90a code (wgmma) loads on compute capability 9.0 only
        return fail(std::string("device '") + prop.name + "' is sm_" + std::to_string(prop.major) + std::to_string(prop.minor) +
                    "; this library is built for sm_90a (H100) only");
    return 0;
}

// Kernel-class timing for bench.py: enable, run, then read a JSON object
// {"gemm": {"launches": n, "ms": t, "work": flops_or_bytes}, ...}.  Reading synchronises the device.
extern "C" int nb200_profile_enable(int on) {
    std::lock_guard<std::mutex> lk(g_prof_mu);
    for (auto& r : g_prof_recs) { g_prof_pool.push_back(r.a); g_prof_pool.push_back(r.b); }
    g_prof_recs.clear();
    g_prof_enabled.store(on ? 1 : 0);
    return 0;
}

extern "C" int nb200_profile_report(char* buf, size_t cap) {
    NB_CHECK(buf && cap > 0, "null buffer");
    NB_CUDA(cudaDeviceSynchronize());
    std::lock_guard<std::mutex> lk(g_prof_mu);
    double ms[PC_COUNT] = {0}, work[PC_COUNT] = {0}, floor_ms[PC_COUNT] = {0}, bytes[PC_COUNT] = {0};
    long n[PC_COUNT] = {0};
    for (auto& r : g_prof_recs) {
        float t = 0.f;
        if (cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess) {
            ms[r.cat] += t; work[r.cat] += r.work; n[r.cat]++;
            // per-launch traffic-mix HBM floor: max((R+W)/copy, W/write_only, R/read_only)
            double f = (r.rb + r.wb) / g_bw_copy;
            if (r.wb / g_bw_write > f) f = r.wb / g_bw_write;
            if (r.rb / g_bw_read > f) f = r.rb / g_bw_read;
            floor_ms[r.cat] += f * 1e3;
            bytes[r.cat] += r.rb + r.wb;
        }
    }
    std::string s = "{";
    bool first = true;
    for (int c = 0; c < PC_COUNT; ++c) {
        if (!n[c]) continue;
        char tmp[256];
        snprintf(tmp, sizeof(tmp), "%s\"%s\": {\"launches\": %ld, \"ms\": %.6f, \"work\": %.6e, \"hbm_bytes\": %.6e, \"hbm_floor_ms\": %.6f}",
                 first ? "" : ", ", kCatNames[c], n[c], ms[c], work[c], bytes[c], floor_ms[c]);
        s += tmp;
        first = false;
    }
    s += "}";
    NB_CHECK(s.size() + 1 <= cap, "buffer too small");
    memcpy(buf, s.c_str(), s.size() + 1);
    return 0;
}

// Per-launch records of the current profile (one CSV line per timed launch: class,ms,work,read_bytes,write_bytes);
// a per-launch roofline table is built from them.  Synchronises the device.
extern "C" int nb200_profile_dump(char* buf, size_t cap) {
    NB_CHECK(buf && cap > 0, "null buffer");
    NB_CUDA(cudaDeviceSynchronize());
    std::lock_guard<std::mutex> lk(g_prof_mu);
    std::string s;
    for (auto& r : g_prof_recs) {
        float t = 0.f;
        if (cudaEventElapsedTime(&t, r.a, r.b) != cudaSuccess) continue;
        char tmp[160];
        snprintf(tmp, sizeof(tmp), "%s,%.6f,%.6e,%.6e,%.6e\n", kCatNames[r.cat], t, r.work, r.rb, r.wb);
        s += tmp;
    }
    NB_CHECK(s.size() + 1 <= cap, "buffer too small");
    memcpy(buf, s.c_str(), s.size() + 1);
    return 0;
}

// Launch recorder: a non-zero mask (REC_GEMMS | REC_AUX | REC_CONV | REC_STEREO | REC_WARP | REC_DEPTH bits, common.cuh) clears the record and starts appending
// the kinds it selects, 0 stops (the record stays readable).  Host only: a launch made while it is off costs one relaxed
// atomic load.
extern "C" int nb200_record_launches(int on) {
    NB_CHECK((on & ~(REC_GEMMS | REC_AUX | REC_CONV | REC_STEREO | REC_WARP | REC_DEPTH)) == 0, "unknown recorder bits");
    std::lock_guard<std::mutex> lk(g_rec_mu);
    if (on) g_rec.clear();
    g_rec_enabled.store(on);
    return 0;
}

static int copy_record(const std::string& s, char* buf, size_t cap) {
    NB_CHECK(buf && cap > 0, "null buffer");
    NB_CHECK(s.size() + 1 <= cap, "buffer too small: " + std::to_string(s.size() + 1) + " bytes needed");
    memcpy(buf, s.c_str(), s.size() + 1);
    return 0;
}

// One line per recorded launch, `kind,name=value,...` (the kinds: see the header).
extern "C" int nb200_recorded_launches_named(char* buf, size_t cap) {
    std::lock_guard<std::mutex> lk(g_rec_mu);
    return copy_record(g_rec, buf, cap);
}

// The same lines without the names, `kind,value,...`: the positional form this entry point has always returned.
extern "C" int nb200_recorded_launches(char* buf, size_t cap) {
    std::lock_guard<std::mutex> lk(g_rec_mu);
    std::string s;
    bool in_name = false;   // names and values hold neither ',' nor '='
    for (const char c : g_rec) {
        if (in_name) {
            in_name = c != '=';
            continue;
        }
        s += c;
        in_name = c == ',';
    }
    return copy_record(s, buf, cap);
}
