// basis.cuh — observables in a per-qubit basis (ExpVarUnitaryAll, reference src/qinterface/qinterface.cpp:478-540) as one
// read-only sweep.
//
// The reference applies a basis gate A_p to each listed qubit q_p, runs the Floats moments query and applies the gates again:
// five state passes, two of them writes.  Here, with K the listed qubits (ascending) and E the others, every environment
// index e owns the block v_e[r] = psi[dep_K(r) | dep_E(e)] of 2^k amplitudes, and the sweep transforms each block in shared
// memory, phi_e = (x)_p A_p v_e, and sums |phi|^2 (1, w - c, (w - c)^2) with the Floats-form weight w of the block index:
//   * blocks are indexed in ASCENDING listed-qubit order (block bit b = the b-th smallest listed qubit); the host permutes the
//     caller's matrices and weights to that order, which is all a relabelling of the tensor factors needs;
//   * a CTA stages a slab of 2^12 amplitudes (min(2^n)) as double2: one block at k = 12, 2^(12 - k) blocks below.  The slab
//     position of (block c, row r) is c 2^k + r.  Global loads are 16 bytes; consecutive load units walk the block rows when
//     qubit 0 is listed (an fp32 chunk is rows 2r, 2r + 1) and the environment columns when it is not (an fp32 chunk is columns
//     2c, 2c + 1).  The one layout where an fp32 chunk straddles two slabs (k = 12 < n, qubit 0 not listed) loads 8-byte
//     amplitudes instead;
//   * the k butterflies run in rounds of up to 3 block bits: each thread holds 8 values in registers at a time, applies the
//     round's butterflies there and writes back, so k = 12 costs 4 shared-memory round trips, not 12.  The last round accumulates
//     instead of writing back.  Every product and sum is in double; the slab is XOR-swizzled so that no round has a
//     shared-memory bank conflict;
//   * the state is read once and never written; each CTA adds one set of partials with one atomic per output.
// Included by b200sv.cu (same translation unit as the other kernels).
#pragma once

#include <algorithm>
#include <vector>

namespace b200sv {

static const int BASIS_SLAB_LOG = 12; // amplitudes per slab: 2^12 double2 = 64 KB, one block at k = B200SV_BASIS_MAX_QUBITS
static const int BASIS_THREADS = 256;
static const int BASIS_ROUND = 3;                                    // block bits per butterfly round
static const int BASIS_VPT = 1 << BASIS_ROUND;                       // values per thread and pass
static const int BASIS_PASSES = (1 << BASIS_SLAB_LOG) / (BASIS_THREADS * BASIS_VPT); // passes per round (2)
static const int BASIS_UPT = (1 << BASIS_SLAB_LOG) / BASIS_THREADS;  // amplitudes per thread and slab (16)

struct BasisArgs {
    int k;          // listed qubits, ascending in keptLow
    int logS;       // amplitudes per slab: 2^logS = min(2^12, 2^n)
    int unitLog;    // load units per slab (amplitudes, or fp32 chunks when paired)
    int pairStride; // paired fp32 chunks: slab distance of a chunk's second amplitude (1 when qubit 0 is listed, else 2^k)
    uint64_t slabs; // 2^(n - logS)
    uint64_t keptLow[B200SV_BASIS_MAX_QUBITS]; // 2^K[b] - 1: the slab base inserts a zero bit at each listed qubit
    int unitAmp[BASIS_SLAB_LOG];               // bit j of a slab's load-unit index -> amplitude index bit
    int unitSlab[BASIS_SLAB_LOG];              // ... -> slab position bit
    double mats[8 * B200SV_BASIS_MAX_QUBITS];  // A for block bit b: m00, m01, m10, m11 (re, im), ascending order
    double weights[2 * B200SV_BASIS_MAX_QUBITS];
    double center;
};

// slab position -> shared-memory slot: XOR the low 3 bits with the other 3-bit digits.  Any 8 accesses whose positions differ in
// 3 consecutive bits only (a quarter-warp of 16-byte accesses in every layout below) land in 8 distinct bank groups.
__device__ __forceinline__ int basis_slot(int s) { return s ^ (((s >> 3) ^ (s >> 6) ^ (s >> 9)) & 7); }

__device__ __forceinline__ double2 cmul_add(double2 a, double2 u, double2 b, double2 v)
{
    return make_double2(fma(a.x, u.x, fma(-a.y, u.y, fma(b.x, v.x, -b.y * v.y))),
        fma(a.x, u.y, fma(a.y, u.x, fma(b.x, v.y, b.y * v.x))));
}

// One butterfly round over block bits lo .. lo + G - 1, in BASIS_PASSES passes of BASIS_VPT values per thread.  Value v of a
// pass: its low G bits are the round's block bits, its high bits pick one of the pass's BASIS_VPT / 2^G groups.  LAST:
// accumulate the moments instead of writing back.
template <int G, bool LAST>
__device__ __forceinline__ void basis_round(double2* sm, const double* mats, const double* wLo, const double* wHi, int lo, int k,
    double center, double& s0, double& s1, double& s2)
{
    constexpr int GPP = BASIS_VPT >> G; // groups per pass
#pragma unroll 1
    for (int pass = 0; pass < BASIS_PASSES; ++pass) {
        int pos[BASIS_VPT];
        double2 r[BASIS_VPT];
#pragma unroll
        for (int v = 0; v < BASIS_VPT; ++v) {
            // group j of the slab (of 2^12 / 2^G) with G zero bits inserted at lo, then the value's round bits
            const int j = threadIdx.x + BASIS_THREADS * (pass * GPP + (v >> G));
            pos[v] = ((j >> lo) << (lo + G)) | (j & ((1 << lo) - 1)) | ((v & ((1 << G) - 1)) << lo);
            r[v] = sm[basis_slot(pos[v])];
        }
#pragma unroll
        for (int h = 0; h < G; ++h) {
            const double* m = mats + 8 * (lo + h);
            const double2 a00 = make_double2(m[0], m[1]), a01 = make_double2(m[2], m[3]);
            const double2 a10 = make_double2(m[4], m[5]), a11 = make_double2(m[6], m[7]);
#pragma unroll
            for (int v = 0; v < BASIS_VPT; ++v) {
                if (!(v & (1 << h))) {
                    const double2 u = r[v], w = r[v | (1 << h)];
                    r[v] = cmul_add(a00, u, a01, w);
                    r[v | (1 << h)] = cmul_add(a10, u, a11, w);
                }
            }
        }
        if (!LAST) {
#pragma unroll
            for (int v = 0; v < BASIS_VPT; ++v) {
                sm[basis_slot(pos[v])] = r[v];
            }
            continue;
        }
        const int rowMask = (1 << k) - 1;
#pragma unroll
        for (int v = 0; v < BASIS_VPT; ++v) {
            const int row = pos[v] & rowMask;
            const double p = fma(r[v].x, r[v].x, r[v].y * r[v].y);
            const double d = wLo[row & 63] * wHi[row >> 6] - center;
            const double pd = p * d;
            s0 += p;
            s1 += pd;
            s2 += pd * d;
        }
    }
}

template <int G>
__device__ __forceinline__ void basis_round_at(bool last, double2* sm, const double* mats, const double* wLo, const double* wHi,
    int lo, int k, double center, double& s0, double& s1, double& s2)
{
    if (last) {
        basis_round<G, true>(sm, mats, wLo, wHi, lo, k, center, s0, s1, s2);
    } else {
        basis_round<G, false>(sm, mats, wLo, wHi, lo, k, center, s0, s1, s2);
    }
}

// out[0..2] += (sum |phi|^2, sum |phi|^2 (w - c), sum |phi|^2 (w - c)^2) over the slabs blockIdx.x, + gridDim.x, ...
// PAIR (fp32 only): a load unit is a 16-byte chunk of two amplitudes that differ in qubit 0.
template <typename R, bool PAIR>
__global__ void __launch_bounds__(BASIS_THREADS, 2) k_moments_basis(const void* __restrict__ amps, const __grid_constant__ BasisArgs a, double* out)
{
    constexpr bool F32 = sizeof(R) == 4;
    constexpr int UPT = (PAIR ? BASIS_UPT / 2 : BASIS_UPT); // load units per thread and slab
    typedef typename std::conditional<F32, typename std::conditional<PAIR, float4, float2>::type, double2>::type V;
    extern __shared__ __align__(16) unsigned char basisSmem[];
    double2* sm = reinterpret_cast<double2*>(basisSmem);
    double* mats = reinterpret_cast<double*>(sm + (1 << BASIS_SLAB_LOG));
    double* wLo = mats + 8 * B200SV_BASIS_MAX_QUBITS; // w = wLo[row & 63] wHi[row >> 6]
    double* wHi = wLo + 64;
    uint64_t* xAmp = reinterpret_cast<uint64_t*>(wHi + 64); // amplitude / slab bits of the unit-index bits above the thread's
    int* xSlab = reinterpret_cast<int*>(xAmp + BASIS_UPT);
    const int t = threadIdx.x;
    const int S = 1 << a.logS, units = 1 << a.unitLog, nbLog = a.logS - a.k;

    for (int i = t; i < 8 * a.k; i += BASIS_THREADS) {
        mats[i] = a.mats[i];
    }
    if (t < 64) {
        double lo = 1.0, hi = 1.0;
        for (int b = 0; b < 6; ++b) {
            const int bit = (t >> b) & 1;
            if (b < a.k) {
                lo *= a.weights[2 * b + bit];
            }
            if (b + 6 < a.k) {
                hi *= a.weights[2 * (b + 6) + bit];
            }
        }
        wLo[t] = lo;
        wHi[t] = hi;
    }
    if (t < UPT) {
        uint64_t am = 0U;
        int sl = 0;
        for (int j = 8; j < a.unitLog; ++j) {
            if (((t << 8) >> j) & 1) {
                am |= 1ULL << a.unitAmp[j];
                sl |= 1 << a.unitSlab[j];
            }
        }
        xAmp[t] = am;
        xSlab[t] = sl;
    }
    // a slab smaller than the shared buffer (n < 12): the slots past it stay zero, so every round can treat all 16 values alike
    for (int i = S + t; i < (1 << BASIS_SLAB_LOG); i += BASIS_THREADS) {
        sm[i] = make_double2(0.0, 0.0);
    }
    uint64_t tAmp = 0U;
    int tSlab = 0;
    for (int j = 0; j < 8 && j < a.unitLog; ++j) {
        if ((t >> j) & 1) {
            tAmp |= 1ULL << a.unitAmp[j];
            tSlab |= 1 << a.unitSlab[j];
        }
    }

    const V* __restrict__ p = reinterpret_cast<const V*>(amps);
    double s0 = 0, s1 = 0, s2 = 0;
    for (uint64_t slab = blockIdx.x; slab < a.slabs; slab += gridDim.x) {
        __syncthreads(); // tables written / the previous slab consumed
        uint64_t base = slab << nbLog; // first environment index of the slab, deposited on the environment qubits
        for (int b = 0; b < a.k; ++b) {
            const uint64_t lo = base & a.keptLow[b];
            base = ((base ^ lo) << 1) | lo;
        }
        // two halves of UPT / 2 loads in flight per thread: within the 128 registers of two CTAs per SM
#pragma unroll 1
        for (int half = 0; half < 2; ++half) {
            V v[UPT / 2];
#pragma unroll
            for (int i = 0; i < UPT / 2; ++i) {
                const int x = half * (UPT / 2) + i;
                v[i] = V{};
                if (t + x * BASIS_THREADS < units) {
                    v[i] = p[(base | tAmp | xAmp[x]) >> (PAIR ? 1 : 0)];
                }
            }
#pragma unroll
            for (int i = 0; i < UPT / 2; ++i) {
                const int x = half * (UPT / 2) + i;
                if (t + x * BASIS_THREADS < units) {
                    const int s = tSlab | xSlab[x];
                    if constexpr (PAIR) {
                        sm[basis_slot(s)] = make_double2((double)v[i].x, (double)v[i].y);
                        sm[basis_slot(s + a.pairStride)] = make_double2((double)v[i].z, (double)v[i].w);
                    } else {
                        sm[basis_slot(s)] = make_double2((double)v[i].x, (double)v[i].y);
                    }
                }
            }
        }
        for (int lo = 0; lo < a.k; lo += BASIS_ROUND) {
            __syncthreads();
            const int g = min(BASIS_ROUND, a.k - lo);
            const bool last = lo + BASIS_ROUND >= a.k;
            switch (g) {
            case 1:
                basis_round_at<1>(last, sm, mats, wLo, wHi, lo, a.k, a.center, s0, s1, s2);
                break;
            case 2:
                basis_round_at<2>(last, sm, mats, wLo, wHi, lo, a.k, a.center, s0, s1, s2);
                break;
            default:
                basis_round_at<3>(last, sm, mats, wLo, wHi, lo, a.k, a.center, s0, s1, s2);
                break;
            }
        }
    }
    block_atomic_add(s0, out);
    block_atomic_add(s1, out + 1);
    block_atomic_add(s2, out + 2);
}

static const size_t BASIS_SMEM = ((size_t)16 << BASIS_SLAB_LOG) + 8 * B200SV_BASIS_MAX_QUBITS * sizeof(double) +
    128 * sizeof(double) + BASIS_UPT * (sizeof(uint64_t) + sizeof(int));

// One basis sweep (arguments validated; the state is non-zero and flushed; 1 <= k <= n).  out[0..2] = S0, S1, S2.
static int launch_moments_basis(State* s, int k, const int* bits, const double* mats8, const double* weights, double center,
    double* out)
{
    const int n = s->nq;
    BasisArgs a{};
    a.k = k;
    a.center = center;
    std::vector<int> ord(k); // ord[b] = the caller's index of the b-th smallest listed qubit
    for (int p = 0; p < k; ++p) {
        ord[p] = p;
    }
    std::sort(ord.begin(), ord.end(), [&](int x, int y) { return bits[x] < bits[y]; });
    uint64_t listed = 0U;
    for (int b = 0; b < k; ++b) {
        const int q = bits[ord[b]];
        listed |= 1ULL << q;
        a.keptLow[b] = (1ULL << q) - 1U;
        std::copy(mats8 + 8 * ord[b], mats8 + 8 * ord[b] + 8, a.mats + 8 * b);
        a.weights[2 * b] = weights[2 * ord[b]];
        a.weights[2 * b + 1] = weights[2 * ord[b] + 1];
    }
    a.logS = std::min(n, BASIS_SLAB_LOG);
    a.slabs = 1ULL << (n - a.logS);
    const int nbLog = a.logS - k;

    // the bits of a slab: block rows (slab bit b <-> listed qubit K[b]) and environment columns (slab bit k + j <-> the j-th
    // lowest other qubit), ordered so that consecutive load units are consecutive in memory as far as the layout allows
    std::vector<std::pair<int, int>> rows, cols; // (amplitude bit, slab bit)
    for (int b = 0; b < k; ++b) {
        rows.push_back({bits[ord[b]], b});
    }
    for (int q = 0; q < n && (int)cols.size() < nbLog; ++q) {
        if (!((listed >> q) & 1U)) {
            cols.push_back({q, k + (int)cols.size()});
        }
    }
    const bool rowsFast = (listed & 1U) != 0;
    std::vector<std::pair<int, int>> unitBits = rowsFast ? rows : cols;
    unitBits.insert(unitBits.end(), rowsFast ? cols.begin() : rows.begin(), rowsFast ? cols.end() : rows.end());
    // fp32: pair the two amplitudes of a 16-byte chunk (qubit 0, the first unit bit) unless qubit 0 is outside the slab
    const bool pair = s->prec == 32 && unitBits[0].first == 0;
    if (pair) {
        a.pairStride = 1 << unitBits[0].second;
        unitBits.erase(unitBits.begin());
    }
    a.unitLog = (int)unitBits.size();
    for (int j = 0; j < a.unitLog; ++j) {
        a.unitAmp[j] = unitBits[j].first;
        a.unitSlab[j] = unitBits[j].second;
    }

    return with_prec(s, [&](auto r) {
        using R = decltype(r);
        void (*kern)(const void*, BasisArgs, double*) = pair ? k_moments_basis<R, sizeof(R) == 4> : k_moments_basis<R, false>;
        SV_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BASIS_SMEM));
        int perSm = 2;
        SV_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, kern, BASIS_THREADS, BASIS_SMEM));
        const uint64_t want = (uint64_t)sm_count(s->dev) * std::max(perSm, 1);
        const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(want, a.slabs));
        SV_TRY(scratch_reduce(s, 3, [&] { kern<<<grid, BASIS_THREADS, BASIS_SMEM, s->stream>>>(s->amps, a, s->d_scratch); }));
        memcpy(out, s->h_scratch, 3 * sizeof(double));
        return B200SV_OK;
    });
}

} // namespace b200sv
