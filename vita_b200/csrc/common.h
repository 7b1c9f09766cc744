// Host-side helpers shared by all translation units of libvita_b200.so.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>
#include <string>
#include <utility>

#include "../../include/vita_b200.h"

namespace vita {

void set_last_error(const std::string& msg);
int num_sms();

// Returns VITA_OK or records the CUDA error text and returns VITA_ERR_CUDA.
int check_cuda(cudaError_t e, const char* what);
int check_launch(const char* what);

#define VITA_REQUIRE(cond, msg)                                                   \
    do {                                                                          \
        if (!(cond)) {                                                            \
            ::vita::set_last_error(std::string(__func__) + ": " + (msg));         \
            return VITA_ERR_INVALID;                                              \
        }                                                                         \
    } while (0)

#define BF16C(p) static_cast<const __nv_bfloat16*>(p)

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// cuTensorMapEncodeTiled resolved through the runtime (no link-time libcuda dependency).
// dims/strides innermost-first; strides in bytes for dims 1..rank-1.
int make_tensor_map_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides,
                         const uint32_t* box, bool swizzle128);

// Programmatic dependent launch (PDL) for the decode chain: kernel N+1 may start (and prefetch weights) while kernel
// N drains; it calls griddepcontrol.wait before touching anything N produced.  Option "pdl" (VITA_B200_PDL).
bool use_pdl();
int option(const char* name);   // tunables table in api.cu (env default, vita_set_option override)

template <typename... KArgs, typename... Args>
inline cudaError_t launch_chain(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                Args&&... args) {
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = use_pdl() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kern, std::forward<Args>(args)...);
}


// Decode-chain completion counters (an accelerator for the programmatic-launch chain, never needed for correctness):
// every kernel of a bs = 1 decode step owns one monotonically increasing 64-bit counter that each of its CTAs bumps
// after its last store; the successor polls it (target = step serial x arrivals per launch) instead of sitting in
// griddepcontrol.wait, which returns ~3.5 us after the predecessor's last CTA has exited (grid teardown + flush).
// A poll that does not succeed within a bounded number of tries falls back to griddepcontrol.wait.
struct ChainArgs {
    const unsigned long long* serial;     // step serial (bumped by decode_embed); nullptr = protocol off
    const unsigned long long* wait_cnt;   // predecessor's counter, nullptr = first kernel of the chain
    unsigned long long* done_cnt;         // this kernel's counter
    int wait_arrivals;                    // arrivals per launch of the predecessor
};
ChainArgs chain_next(int arrivals);       // next link for a chain-capable launch (all-null when no chain is open)

// Optional timeline instrumentation (build with -DVITA_TRACE): the decode-chain kernels stamp %globaltimer at a few
// points into one 32-word record per launch; scripts/decode_trace.py turns the records into a per-kernel timeline.
#ifdef VITA_TRACE
unsigned long long* trace_next_record();   // device pointer for the next launch, or nullptr when tracing is off
#define VITA_TRACE_PARAM , unsigned long long* trace
#define VITA_TRACE_ARG , trace_next_record()
#else
#define VITA_TRACE_PARAM
#define VITA_TRACE_ARG
#endif

}  // namespace vita
