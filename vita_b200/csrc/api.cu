// Library plumbing: error reporting, launch accounting, device query, TMA descriptor encoding.
#include <atomic>
#include <cstdlib>
#include <mutex>

#include "common.h"

namespace vita {

static thread_local std::string g_last_error;
static std::atomic<long long> g_launches{0};

void set_last_error(const std::string& msg) { g_last_error = msg; }

int check_cuda(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return VITA_OK;
    set_last_error(std::string(what) + ": " + cudaGetErrorString(e));
    return VITA_ERR_CUDA;
}

int check_launch(const char* what) {
    g_launches.fetch_add(1, std::memory_order_relaxed);
    return check_cuda(cudaGetLastError(), what);
}

int num_sms() {
    static int cached = -1;
    if (cached < 0) {
        int dev = 0, n = 0;
        if (cudaGetDevice(&dev) != cudaSuccess ||
            cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) {
            (void)cudaGetLastError();
            return 0;
        }
        cached = n;
    }
    return cached;
}

// Tunables: default <- environment variable (read once) <- vita_set_option().
struct Option {
    const char* name;
    const char* env;
    int def;
    std::atomic<int> value;
};
static Option g_options[] = {
    // programmatic dependent launch for the decode chain (trigger after each CTA's last weight load)
    {"pdl", "VITA_B200_PDL", 1, {-1}},
    // tensor-core decode kernels: weight tiles per CTA prefetched into L2 behind the shared-memory ring
    {"tc_l2_ahead", "VITA_B200_TC_L2AHEAD", 0, {-1}},
    // paged decode attention: fetch the cached K/V rows ahead of the dependency wait (needs chain_wait)
    {"attn_early", "VITA_B200_ATTN_EARLY", 1, {-1}},
    // paged decode attention: split partials as tagged 64-bit words collected by split 0 (no fence / ticket)
    {"attn_tagged", "VITA_B200_ATTN_TAGGED", 1, {-1}},
    // decode-chain kernels ask for the maximum shared-memory carve-out
    {"smem_carveout_max", "VITA_B200_SMEM_CARVEOUT_MAX", 0, {-1}},
    // chain kernels wait for their predecessor before they trigger their successor: when kernel N+1 starts, kernel
    // N-1 has completed (what attn_early relies on)
    {"chain_wait", "VITA_B200_CHAIN_WAIT", 1, {-1}},
    // tensor-core gate|up kernel: all 256 threads share the router dot products
    {"tc_wide_route", "VITA_B200_TC_WIDE_ROUTE", 1, {-1}},
    // tensor-core decode kernels: weight tiles still to be issued by a CTA when it triggers the dependent launch
    {"tc_trigger_lead", "VITA_B200_TC_TRIGGER_LEAD", 0, {-1}},
    // tensor-core decode kernels: producer / MMA / x-writer threads that cannot proceed before the predecessor has completed
    // wait in hardware (griddepcontrol.wait) instead of spinning on their mbarriers next to the predecessor's threads
    {"tc_park", "VITA_B200_TC_PARK", 1, {-1}},
    // tensor-core decode kernels: pull norm / router weights into L2 ahead of the dependency wait
    {"tc_prefetch_consts", "VITA_B200_TC_PREFETCH_CONSTS", 1, {-1}},
    // decode chain: per-kernel completion counters polled by the successor instead of griddepcontrol.wait
    {"chain_counters", "VITA_B200_CHAIN_COUNTERS", 0, {-1}},
    // FlashAttention: column chunks (of 4 per key tile) whose exp2 runs as a polynomial on the FMA pipe (relative error
    // 7.5e-5) instead of MUFU ex2.  Off: on an H100 80GB HBM3 (700 W) one chunk gains 3 % on the attention kernel alone
    // (289 vs 298 us, causal GQA 32/8 x 128 at S = 4096; 134 vs 137 us, ViT 16 x 64 at S = 1025, batch 8), about 0.2 ms
    // of a 145 ms prefill, and the exact exponent keeps the probabilities at fp32 accuracy before their bf16 rounding.
    {"fa_poly", "VITA_B200_FA_POLY", 0, {-1}},
};

int option(const char* name) {
    for (Option& o : g_options) {
        if (std::string(o.name) != name) continue;
        int v = o.value.load(std::memory_order_relaxed);
        if (v < 0) {
            const char* e = getenv(o.env);
            v = (e != nullptr && e[0] != '\0') ? atoi(e) : o.def;
            if (v < 0) v = 0;
            o.value.store(v, std::memory_order_relaxed);
        }
        return v;
    }
    return 0;
}

bool use_pdl() { return option("pdl") != 0; }

// chain state of the calling host thread: set by vita_chain_begin, consumed link by link by the chain-capable launches
struct ChainState {
    unsigned long long* mem = nullptr;   // [0] = step serial, [1 + i] = counter of link i
    long long n = 0, next = 0;
    int prev_arrivals = 0;
};
static thread_local ChainState g_chain;

ChainArgs chain_next(int arrivals) {
    ChainArgs a{nullptr, nullptr, nullptr, 0};
    ChainState& c = g_chain;
    if (c.mem == nullptr || c.next >= c.n || !option("chain_counters")) return a;
    a.serial = c.mem;
    a.done_cnt = c.mem + 1 + c.next;
    if (c.next > 0) {
        a.wait_cnt = c.mem + c.next;
        a.wait_arrivals = c.prev_arrivals;
    }
    c.prev_arrivals = arrivals;
    ++c.next;
    return a;
}

#ifdef VITA_TRACE
static unsigned long long* g_trace_base = nullptr;
static long long g_trace_records = 0, g_trace_serial = 0;
unsigned long long* trace_next_record() {
    if (!g_trace_base || g_trace_records <= 0) return nullptr;
    return g_trace_base + ((g_trace_serial++) % g_trace_records) * 32;
}
#endif

}  // namespace vita

extern "C" int vita_set_option(const char* name, int64_t value) {
    VITA_REQUIRE(name != nullptr && value >= 0, "vita_set_option: name and a non-negative value are required");
    for (vita::Option& o : vita::g_options) {
        if (std::string(o.name) == name) {
            o.value.store(static_cast<int>(value), std::memory_order_relaxed);
            return VITA_OK;
        }
    }
    vita::set_last_error(std::string("vita_set_option: unknown option '") + name + "'");
    return VITA_ERR_INVALID;
}

extern "C" int64_t vita_get_option(const char* name) { return name ? vita::option(name) : 0; }

extern "C" int vita_chain_begin(uint64_t* mem, int64_t n_links) {
    VITA_REQUIRE(mem != nullptr && n_links > 0, "vita_chain_begin: counter memory ([1 + n_links] x 8 bytes) required");
    vita::g_chain.mem = reinterpret_cast<unsigned long long*>(mem);
    vita::g_chain.n = n_links;
    vita::g_chain.next = 0;
    vita::g_chain.prev_arrivals = 0;
    return VITA_OK;
}
extern "C" int vita_chain_end(void) {
    vita::g_chain = vita::ChainState{};
    return VITA_OK;
}

#ifdef VITA_TRACE
// instrumentation builds only: records = number of 32-word records in buf; restarts the launch serial
extern "C" int vita_debug_trace(void* buf, int64_t records) {
    vita::g_trace_base = static_cast<unsigned long long*>(buf);
    vita::g_trace_records = records;
    vita::g_trace_serial = 0;
    return VITA_OK;
}
#endif

namespace vita {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(p);
        else
            (void)cudaGetLastError();
    });
    return fn;
}

int make_tensor_map_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                         const uint32_t* box, bool swizzle128) {
    EncodeTiledFn fn = get_encode_fn();
    if (!fn) {
        set_last_error("cuTensorMapEncodeTiled is not available (no CUDA driver?)");
        return VITA_ERR_CUDA;
    }
    cuuint64_t gdims[5];
    cuuint64_t gstrides[4];
    cuuint32_t gbox[5], estr[5];
    for (int i = 0; i < rank; ++i) {
        gdims[i] = dims[i];
        gbox[i] = box[i];
        estr[i] = 1;
    }
    for (int i = 0; i + 1 < rank; ++i) gstrides[i] = strides[i];
    const CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, static_cast<cuuint32_t>(rank), const_cast<void*>(base),
                          gdims, gstrides, gbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                          swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                          CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
        set_last_error("cuTensorMapEncodeTiled failed with CUresult " + std::to_string(static_cast<int>(r)));
        return VITA_ERR_CUDA;
    }
    return VITA_OK;
}

}  // namespace vita

extern "C" int vita_version(void) { return 100; }
extern "C" const char* vita_last_error(void) { return vita::g_last_error.c_str(); }
extern "C" int vita_num_sms(void) { return vita::num_sms(); }
extern "C" int64_t vita_launch_count(int reset) {
    const long long v = vita::g_launches.load();
    if (reset) vita::g_launches.store(0);
    return v;
}
