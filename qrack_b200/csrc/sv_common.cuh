// sv_common.cuh — shared declarations of the state-vector core (internal; the public ABI is include/b200sv.h).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/b200sv.h"

namespace b200sv {

// ---------------------------------------------------------------------------------------------------------
// complex helpers: amplitudes are interleaved (re,im) = float2 / double2 (reference statevector.hpp:94)
// ---------------------------------------------------------------------------------------------------------
template <typename R> struct Cx;
template <> struct Cx<float> {
    typedef float2 type;
};
template <> struct Cx<double> {
    typedef double2 type;
};

template <typename R> __host__ __device__ __forceinline__ typename Cx<R>::type mk(R re, R im)
{
    typename Cx<R>::type c;
    c.x = re;
    c.y = im;
    return c;
}
template <typename C> __device__ __forceinline__ C cmul(const C a, const C b)
{
    C r;
    r.x = a.x * b.x - a.y * b.y;
    r.y = a.x * b.y + a.y * b.x;
    return r;
}
// r = a*x + b*y
template <typename C> __device__ __forceinline__ C cmad2(const C a, const C x, const C b, const C y)
{
    C r;
    r.x = a.x * x.x - a.y * x.y + b.x * y.x - b.y * y.y;
    r.y = a.x * x.y + a.y * x.x + b.x * y.y + b.y * y.x;
    return r;
}
template <typename C> __device__ __forceinline__ auto cnorm(const C a) -> decltype(a.x) { return a.x * a.x + a.y * a.y; }

// 2x2 matrix passed by value in kernel params (row-major m0 m1 / m2 m3)
template <typename R> struct Mat2 {
    typename Cx<R>::type m[4];
};

// sorted qubit powers for the "insert zero bits" index map (reference parallel_for.cpp:118-149, qengine.cu:89-107)
struct PowList {
    int n;
    uint64_t low[64]; // low[k] = pow_k - 1
};

__host__ __device__ __forceinline__ uint64_t push_apart(uint64_t i, const PowList& p)
{
    for (int k = 0; k < p.n; ++k) {
        const uint64_t lo = i & p.low[k];
        i = ((i ^ lo) << 1) | lo;
    }
    return i;
}

// ---------------------------------------------------------------------------------------------------------
// queued gate (single target qubit + control mask/value), the unit the fused sweep consumes
// ---------------------------------------------------------------------------------------------------------
struct GateOp {
    int target;         // target qubit, or -1 for a pure diagonal "phase on predicate" op
    uint64_t cmask;     // control qubits (bits)
    uint64_t cval;      // required values of the control qubits
    double m[8];        // 2x2 complex, row-major (nrm already folded in)
    int kind;           // 0 general, 1 diagonal (m1=m2=0), 2 anti-diagonal (m0=m3=0)
};

// Pending "pull" re-page (multi-process exchange, b200sv_exchange_pull): the state's content is DEFINED as the exchanged view of
// the ranks' source pages — element i of this rank's new page is element ((i & ~vmask) | rankDep) of the page of the rank named by
// the victim bits of i — and is materialised into `out` by the first sweep of the next flush (k_fused_sweep<..., PULL>), whose
// first pass reads through the peer mappings, or by the plain gather kernel when no sweep follows.  Indices in amplitudes.
struct PullArgs {
    const void* peers[8];
    void* out;
    uint64_t vmask;   // OR of the victim bits
    uint64_t rankDep; // this rank's index bits deposited at the victim positions
    int vb[3];
    int k;
};

struct State {
    int dev = 0;
    int nq = 0;
    int prec = 32;
    void* amps = nullptr; // device buffer (nullptr == the zero state)
    size_t amps_bytes = 0; // size it was allocated with through the state-buffer cache (0: plain cudaMalloc / external)
    bool external = false;
    void* spare = nullptr; // second state-sized buffer kept by the out-of-place QAlu sweeps (ping-pong with amps)
    size_t spare_bytes = 0;
    cudaStream_t stream = nullptr;
    bool ownStream = true;
    double* d_scratch = nullptr; // small device scratch for reductions
    size_t scratch_doubles = 0;
    double* h_scratch = nullptr; // pinned host mirror
    void* d_flush = nullptr;     // L2 flush buffer
    size_t flush_bytes = 0;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, evx = nullptr;
    int fusion = 1;
    std::vector<GateOp> queue;
    bool pullPending = false; // see PullArgs
    PullArgs pull{};
    b200sv_stats stats{};
    // memoised single-qubit marginals: marg[b] = sum |psi_i|^2 over i with bit b set, marg[64] = sum over all i.
    // Filled by ONE sweep on the first Prob(q) after a change; every mutating ABI call clears `margValid`.
    bool margValid = false;
    double marg[65];

    size_t amp_bytes() const { return prec == 32 ? 8 : 16; }
    uint64_t dim() const { return 1ULL << nq; }
};

void set_error(const std::string& msg);
int cuda_fail(cudaError_t e, const char* what);

#define SV_CUDA(call)                                                                                                  \
    do {                                                                                                               \
        cudaError_t e__ = (call);                                                                                      \
        if (e__ != cudaSuccess)                                                                                        \
            return ::b200sv::cuda_fail(e__, #call);                                                                    \
    } while (0)

#define SV_TRY(call)                                                                                                   \
    do {                                                                                                               \
        int r__ = (call);                                                                                              \
        if (r__ != B200SV_OK)                                                                                          \
            return r__;                                                                                                \
    } while (0)

int sm_count(int dev);

// fused.cu
int fused_flush(State* s);
int launch_xmask(State* s, uint64_t mask); // the dedicated XMask permutation sweep (b200sv.cu); does not flush
bool fused_accepts(const State* s, const GateOp& g);
void fused_release(State* s);
int launch_pull_gather(State* s); // the pending pull as a plain gather kernel (b200sv.cu); adopts the out page
int fused_emulate(int n_qubits, int precision, const std::vector<GateOp>& q, void* host_state, const PullArgs* pull = nullptr);
int fused_plan_gates(int n_qubits, int precision, const std::vector<GateOp>& q, int* n_sweeps, int* n_passes, int* n_ops);

} // namespace b200sv

struct b200sv_state : public b200sv::State {};
